"""GPU parity tests of the fused network ops (through the C ABI op program) against torch-CPU fp32 references and the
oracle, in fp32 and bf16 activations.  Bounds: tests/util.py::check_op (fp32 |err| <= 2e-4 * max|ref|, bf16 relative
L2 <= 1e-2 per op) unless a test states its own; the network-level checks are in tests/test_backbones_gpu.py.
"""
import pytest
import torch
import torch.nn.functional as F

from tests.util import DEV, builder, check_op, external, nchw, run_op

pytestmark = pytest.mark.gpu


TC_CASES = [
    # cins, cout, k, stride, H, W, res, relu, out
    ([64], 64, 3, 1, 16, 16, False, True, "act"),        # exactly one tile per image
    ([64], 64, 3, 1, 40, 48, True, True, "act"),         # partial tiles, residual
    ([16], 16, 3, 1, 64, 64, False, True, "act"),        # BK=16 (SW32)
    ([16], 32, 3, 2, 64, 64, False, True, "act"),        # stride 2 (TMA element strides), BK=16
    ([32], 64, 3, 2, 32, 32, False, True, "act"),        # stride 2, BK=32 (SW64)
    ([32], 64, 1, 1, 16, 24, False, False, "act"),       # 1x1, BK=32
    ([128], 256, 3, 2, 32, 32, False, True, "act"),      # stride 2, BN=256
    ([256], 512, 3, 1, 16, 16, True, True, "act"),       # two N tiles
    ([128, 128, 64, 128], 128, 1, 1, 16, 16, False, True, "act"),   # Root: 4 K-slabs
    ([512, 512, 256], 512, 1, 1, 8, 8, False, True, "act"),         # TW=8 tiles
    ([128], 27, 3, 1, 24, 24, False, False, "f32"),      # DCN offset/mask conv: fp32 out, cout 27
    ([64], 256, 3, 1, 32, 32, False, True, "act"),       # head 3x3
    # small-channel 3x3 convs take the SIMT-fed kernel (csrc/net_tc_sp.cu): both strides, partial tiles, residual
    ([16], 16, 3, 1, 21, 37, False, True, "act"),
    ([16], 32, 3, 2, 37, 51, False, True, "act"),
    ([16], 64, 3, 1, 16, 8, True, False, "act"),
    ([32], 32, 3, 1, 40, 24, True, True, "act"),         # HRNet branch-0 block conv with residual
    ([32], 64, 3, 2, 50, 30, False, True, "act"),
    ([32], 32, 3, 2, 33, 17, False, False, "act"),
    ([32], 16, 3, 1, 19, 23, False, True, "act"),
    ([256], 34, 1, 1, 32, 32, False, False, "nchw"),     # head 1x1 -> NCHW fp32 logits (hps)
    ([256], 1, 1, 1, 24, 40, False, False, "nchw"),      # head 1x1 (hm), partial tiles
    ([64], 17, 1, 1, 16, 16, False, True, "nchw"),
]


@pytest.mark.parametrize("cins,cout,k,stride,H,W,res,relu,out", TC_CASES)
def test_conv_tensor_core_path(cins, cout, k, stride, H, W, res, relu, out):
    """wgmma implicit-GEMM conv vs torch fp32 on the same bf16-rounded inputs/weights.
    Tolerance: |err| <= 1e-2 * max|ref| (bf16 output rounding 2^-9 + fp32 accumulation order)."""
    B = 3
    g = torch.Generator().manual_seed(sum(cins) * 7 + cout + k + stride)
    xs = [torch.randn(B, c, H, W, generator=g).bfloat16().float() for c in cins]
    w = (torch.randn(cout, sum(cins), k, k, generator=g) / (sum(cins) * k * k) ** 0.5).bfloat16().float()
    b = torch.randn(cout, generator=g)
    pad = k // 2
    ref = F.conv2d(torch.cat(xs, 1), w, b, stride=stride, padding=pad)
    r = None
    if res:
        r = torch.randn(ref.shape, generator=g).bfloat16().float()
        ref = ref + r
    if relu:
        ref = F.relu(ref)
    pb = builder(B, "bf16", tc=True)
    sx = [external(pb, x, "bf16") for x in xs]
    sr = external(pb, r, "bf16") if res else None
    if out == "nchw":
        dst = pb.output(cout + 3, ref.shape[2], ref.shape[3], "o")
        buf = torch.zeros(B, cout + 3, ref.shape[2], ref.shape[3], device=DEV)
        pb.conv(sx, w.to(DEV), b.to(DEV), stride=stride, pad=pad, relu=relu, out="nchw", dst=dst, ch_off=2)
        assert pb.ops[-1].flags & 8
        plan = pb.build(); plan.bind(torch.zeros(1, device=DEV), {"o": buf})
        plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
        assert buf[:, :2].abs().max().item() == 0 and buf[:, cout + 2:].abs().max().item() == 0
        got = buf[:, 2:cout + 2].cpu()
        err = (got - ref).abs().max().item()
        assert err <= 2e-3 * ref.abs().max().item(), (err, ref.abs().max().item())   # fp32 out: only accumulation order
        return
    y = pb.conv(sx, w.to(DEV), b.to(DEV), stride=stride, pad=pad, relu=relu, res=sr, out=out)
    assert pb.ops[-1].flags & 8, "op was not routed to the tensor-core path"
    got = run_op(pb, y)
    err = (got - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), (err, ref.abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("cins,cout,k,stride,H,W,res,relu", [
    ([16], 16, 3, 1, 20, 24, False, True), ([16], 32, 3, 2, 20, 24, False, True),
    ([64], 64, 3, 1, 17, 13, True, True), ([32], 64, 1, 1, 9, 9, False, False),
    ([64, 64, 32], 128, 1, 1, 10, 12, False, True), ([128], 27, 3, 1, 8, 8, False, False),
    ([256], 34, 1, 1, 8, 8, False, False), ([64], 256, 3, 1, 12, 12, False, True),
    ([512], 512, 3, 1, 4, 4, True, True),
])
def test_conv_op(precision, cins, cout, k, stride, H, W, res, relu):
    B = 2
    g = torch.Generator().manual_seed(sum(cins) + cout + k)
    xs = [torch.randn(B, c, H, W, generator=g) for c in cins]
    if precision == "bf16":
        xs = [x.bfloat16().float() for x in xs]
    w = torch.randn(cout, sum(cins), k, k, generator=g) / (sum(cins) * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    pad = k // 2
    ref = F.conv2d(torch.cat(xs, 1), w, b, stride=stride, padding=pad)
    r = None
    if res:
        r = torch.randn(ref.shape, generator=g)
        if precision == "bf16":
            r = r.bfloat16().float()
        ref = ref + r
    if relu:
        ref = F.relu(ref)
    pb = builder(B, precision, tc=False)
    sx = [external(pb, x, precision) for x in xs]
    sr = external(pb, r, precision) if res else None
    y = pb.conv(sx, w.to(DEV), b.to(DEV), stride=stride, pad=pad, relu=relu, res=sr)
    check_op(run_op(pb, y), ref, precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_conv_nchw_and_f32_outputs(precision):
    B, C, H, W = 2, 32, 6, 10
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, C, H, W, generator=g).bfloat16().float()
    w = torch.randn(5, C, 1, 1, generator=g) * 0.2; b = torch.randn(5, generator=g)
    ref = F.conv2d(x, w, b)
    pb = builder(B, precision, tc=False)
    out = torch.zeros(B, 7, H, W, device=DEV)
    dst = pb.output(7, H, W, "o")
    pb.conv([external(pb, x, precision)], w.to(DEV), b.to(DEV), out="nchw", dst=dst, ch_off=2)
    y32 = pb.conv([external(pb, x, precision)], w.to(DEV), b.to(DEV), out="f32")
    plan = pb.build()
    plan.bind(torch.zeros(1, device=DEV), {"o": out})
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    check_op(out[:, 2:7].cpu(), ref, precision, 2e-3 if precision == "bf16" else None)
    assert out[:, :2].abs().max().item() == 0
    assert plan.tensor(y32).dtype == torch.float32
    check_op(nchw(plan.tensor(y32)), ref, precision, 2e-3 if precision == "bf16" else None)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_stem_maxpool_upadd_ops(precision):
    B = 2
    g = torch.Generator().manual_seed(2)
    # stem 7x7 3->16 on NCHW fp32 input
    x = torch.randn(B, 3, 32, 40, generator=g)
    w = torch.randn(16, 3, 7, 7, generator=g) * 0.1; b = torch.randn(16, generator=g)
    pb = builder(B, precision, tc=False); pb.H, pb.W = 32, 40
    xin = pb.input(3)
    y = pb.stem(xin, w.to(DEV), b.to(DEV), 7, 1, 3, relu=True)
    plan = pb.build(); plan.bind(x.to(DEV), {}); plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    check_op(nchw(plan.tensor(y)), F.relu(F.conv2d(x, w, b, padding=3)), precision)
    # maxpool 2x2/s2 and 3x3/s2/p1
    t = torch.randn(B, 32, 16, 20, generator=g).bfloat16().float()
    for (k, s, p) in ((2, 2, 0), (3, 2, 1)):
        pb = builder(B, precision, tc=False)
        y = pb.maxpool(external(pb, t, precision), k, s, p)
        assert torch.equal(run_op(pb, y), F.max_pool2d(t, k, s, p))
    # depthwise deconv (f = 2 and f = 4) + skip; C = 48 fails the fast kernel's shape condition (generic kernel) and
    # draws from its own generator, so the cases after it see the same data as without it
    for f, C, gen in ((2, 32, g), (4, 32, g), (2, 48, torch.Generator().manual_seed(48))):
        xx = torch.randn(B, C, 6, 7, generator=gen).bfloat16().float()
        ww = torch.rand(C, 1, 2 * f, 2 * f, generator=gen)
        ref_up = F.conv_transpose2d(xx, ww, None, stride=f, padding=f // 2, groups=C)
        skip = torch.randn(ref_up.shape, generator=gen).bfloat16().float()
        pb = builder(B, precision, tc=False)
        y = pb.up_add(external(pb, xx, precision), external(pb, skip, precision), ww.to(DEV))
        check_op(run_op(pb, y), ref_up + skip, precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("ci,co,H,W", [(64, 64, 12, 14), (128, 64, 8, 8), (32, 48, 9, 11)])
def test_dcn_op_matches_oracle(precision, ci, co, H, W):
    from oracle import dcn_ref
    B = 2
    g = torch.Generator().manual_seed(ci + co)
    x = torch.randn(B, ci, H, W, generator=g).bfloat16().float()
    w = torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5; b = torch.randn(co, generator=g)
    ow = torch.randn(27, ci, 3, 3, generator=g) * (1.5 / (ci * 9) ** 0.5); ob = torch.randn(27, generator=g)
    ref = F.relu(dcn_ref.dcn_module_forward(x, w, b, ow, ob))
    pb = builder(B, precision, tc=False)
    y = pb.dcn(external(pb, x, precision), w.to(DEV), b.to(DEV), ow.to(DEV), ob.to(DEV), relu=True)
    # bf16: offsets come from a bf16-input conv -> sampling positions differ slightly
    check_op(run_op(pb, y), ref, precision, 2e-2 if precision == "bf16" else 5e-4)


@pytest.mark.parametrize("ci,co,H,W", [(64, 64, 16, 16), (128, 64, 24, 40), (256, 256, 16, 16), (512, 256, 8, 8), (64, 128, 33, 20)])
def test_dcn_tensor_core_path(ci, co, H, W):
    """wgmma DCN (gather producers write the swizzled A tile) vs the oracle on bf16-rounded data.
    Offsets are large (gain 1.5: many samples out of bounds).  Tolerance: relative L2 <= 1e-2 and
    |err| <= 3e-2 max|ref| (bf16 A-operand rounding after the fp32 bilinear blend, bf16 output)."""
    from oracle import dcn_ref
    B = 2
    g = torch.Generator().manual_seed(ci * 3 + co)
    x = torch.randn(B, ci, H, W, generator=g).bfloat16().float()
    w = (torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5).bfloat16().float(); b = torch.randn(co, generator=g)
    ow = (torch.randn(27, ci, 3, 3, generator=g) * (1.5 / (ci * 9) ** 0.5)).bfloat16().float(); ob = torch.randn(27, generator=g)
    ref = F.relu(dcn_ref.dcn_module_forward(x, w, b, ow, ob))
    pb = builder(B, "bf16", tc=True)
    y = pb.dcn(external(pb, x, "bf16"), w.to(DEV), b.to(DEV), ow.to(DEV), ob.to(DEV), relu=True)
    assert pb.ops[-1].type == 5 and pb.ops[-1].flags & 8, "DCN op was not routed to the tensor-core path"
    got = run_op(pb, y)
    rel = ((got - ref).norm() / ref.norm()).item()
    err = (got - ref).abs().max().item()
    assert rel <= 1e-2 and err <= 3e-2 * ref.abs().max().item(), (rel, err, ref.abs().max().item())


def test_dcn_tensor_core_zero_offset_identity():
    """DCNv2/test.py:31-66 on the wgmma DCN: zero offsets, mask 0.5, identity weights => 2*out == in
    (exact: 0.5*x is representable in bf16)."""
    B, C, H, W = 2, 64, 24, 16
    x = torch.randint(-8, 9, (B, C, H, W), generator=torch.Generator().manual_seed(0)).float()
    w = torch.zeros(C, C, 3, 3)
    for c in range(C):
        w[c, c, 1, 1] = 1.0
    pb = builder(B, "bf16", tc=True)
    y = pb.dcn(external(pb, x, "bf16"), w.to(DEV), torch.zeros(C, device=DEV),
               torch.zeros(27, C, 3, 3, device=DEV), torch.zeros(27, device=DEV), relu=False)
    assert pb.ops[-1].flags & 8
    out = run_op(pb, y)
    assert torch.equal(2 * out, x)


def test_dcn_zero_offset_identity():
    """DCNv2/test.py:31-66 check_zero_offset on the CUDA op: 2 * out == in."""
    B, C, H, W = 2, 16, 10, 12
    x = torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(0))
    w = torch.zeros(C, C, 3, 3)
    for c in range(C):
        w[c, c, 1, 1] = 1.0
    pb = builder(B, "fp32", tc=False)
    y = pb.dcn(external(pb, x, "fp32"), w.to(DEV), torch.zeros(C, device=DEV),
               torch.zeros(27, C, 3, 3, device=DEV), torch.zeros(27, device=DEV), relu=False)
    out = run_op(pb, y)
    assert (2 * out - x).abs().max().item() < 1e-6


@pytest.mark.parametrize("co,stride,H,W", [(16, 1, 48, 40), (16, 1, 21, 37), (64, 2, 64, 96), (64, 2, 38, 50), (16, 2, 32, 32),
                                           (64, 1, 16, 24)])
def test_stem_tensor_core_kernel(co, stride, H, W):
    """csrc/net_stem_tc.cu: 7x7 Cin-3 stem with the im2col built in shared memory + wgmma, vs torch fp32 on
    bf16-rounded image and weights (partial tiles, both strides, both output widths)."""
    B = 3
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, 3, H, W, generator=g).bfloat16().float()
    w = (torch.randn(co, 3, 7, 7, generator=g) * 0.1).bfloat16().float(); b = torch.randn(co, generator=g)
    ref = F.relu(F.conv2d(x, w, b, stride=stride, padding=3))
    pb = builder(B, "bf16", tc=True); pb.H, pb.W = H, W
    y = pb.stem(pb.input(3), w.to(DEV), b.to(DEV), 7, stride, 3, relu=True)
    assert [o.type for o in pb.ops] == [2] and pb.ops[0].flags & 8
    plan = pb.build(); plan.bind(x.to(DEV), {}); plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got = nchw(plan.tensor(y))
    assert got.shape == ref.shape
    err = (got - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item(), (err, ref.abs().max().item())


@pytest.mark.parametrize("mode", ["fp32", "bf16", "bf16tc"])
def test_dense_deconv_lowering(mode):
    """ConvTranspose2d(k4,s2,p1)+BN+ReLU (msra_resnet.py:168-193) lowered to four parity 2x2 convs."""
    from centerpose_b200.archs.resnet import _deconv_bn_relu
    from centerpose_b200.archs.common import StateView
    B, ci, co, H, W = 2, 64, 32, 12, 16
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, ci, H, W, generator=g).bfloat16().float()
    wt = (torch.randn(ci, co, 4, 4, generator=g) / (ci * 4) ** 0.5).bfloat16().float()
    bnp = {"weight": torch.rand(co, generator=g) + 0.5, "bias": torch.randn(co, generator=g) * 0.1,
           "running_mean": torch.randn(co, generator=g) * 0.1, "running_var": torch.rand(co, generator=g) + 0.5}
    ref = F.relu(F.batch_norm(F.conv_transpose2d(x, wt, None, stride=2, padding=1), bnp["running_mean"], bnp["running_var"],
                              bnp["weight"], bnp["bias"], False, 0.0, 1e-5))
    sd = {"d.weight": wt, **{"b." + k: v for k, v in bnp.items()}}
    precision = "fp32" if mode == "fp32" else "bf16"
    pb = builder(B, precision, tc=(mode == "bf16tc"))
    y = _deconv_bn_relu(pb, StateView(sd, "", torch.device(DEV)), external(pb, x, precision), "d", "b")
    if mode == "bf16tc":
        assert all(o.flags & 8 for o in pb.ops)
    check_op(run_op(pb, y), ref, precision, 1.5e-2 if precision == "bf16" else None)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_upsample_add_op_matches_torch(precision):
    """CPB200_OP_UPSAMPLE_ADD (HRNet fuse term): nearest upsample x f + skip (+ReLU); exact in both dtypes up to
    the output rounding.  Also the 3x3 / stride-2 stem (HRNet conv1)."""
    g = torch.Generator().manual_seed(3)
    B, C, H, W = 2, 32, 5, 7
    for f, relu, skip in ((2, True, True), (4, False, True), (8, True, False)):
        xt = torch.randn(B, C, H, W, generator=g).bfloat16().float()
        st = torch.randn(B, C, H * f, W * f, generator=g).bfloat16().float()
        pb = builder(B, precision, tc=False)
        y = pb.upsample_add(external(pb, xt, precision), external(pb, st, precision) if skip else None, f, relu=relu)
        ref = F.interpolate(xt, scale_factor=f, mode="nearest") + (st if skip else 0)
        ref = F.relu(ref) if relu else ref
        check_op(run_op(pb, y), ref, precision)
    img = torch.randn(B, 3, 32, 48, generator=g)
    w = torch.randn(64, 3, 3, 3, generator=g) * 0.2; b = torch.randn(64, generator=g)
    pb = builder(B, precision, tc=False); pb.H, pb.W = 32, 48
    y = pb.stem(pb.input(3), w.to(DEV), b.to(DEV), 3, 2, 1, relu=True)
    plan = pb.build(); plan.bind(img.to(DEV), {})
    plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
    check_op(nchw(plan.tensor(y)), F.relu(F.conv2d(img, w, b, stride=2, padding=1)), precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_mobilenet_ops_match_torch(precision):
    """CPB200_OP_DWCONV / AVGPOOL / SCALE_ADD and the h-swish / h-sigmoid epilogues (mobilenetv3.py:84-147)."""
    from oracle.mobilenet_ref import hsigmoid, hswish
    g = torch.Generator().manual_seed(11)
    B, C, H, W = 2, 48, 13, 18
    x = (torch.randn(B, C, H, W, generator=g) * 2).bfloat16().float()
    for k, stride, act, fn in ((3, 1, "relu", F.relu), (5, 2, "hswish", hswish), (5, 1, None, lambda t: t), (3, 2, "hswish", hswish),
                                (7, 1, "relu", F.relu)):          # 7x7 takes the generic (untiled) kernel
        w = torch.randn(C, 1, k, k, generator=g) * 0.3; b = torch.randn(C, generator=g)
        pb = builder(B, precision, tc=False)
        y = pb.dwconv(external(pb, x, precision), w.to(DEV), b.to(DEV), stride=stride, act=act)
        check_op(run_op(pb, y), fn(F.conv2d(x, w, b, stride=stride, padding=k // 2, groups=C)), precision)
    # global average pool + gate * x + skip
    gate = torch.rand(B, C, 1, 1, generator=g).bfloat16().float(); skip = torch.randn(B, C, H, W, generator=g).bfloat16().float()
    pb = builder(B, precision, tc=False)
    sx = external(pb, x, precision)
    pooled = pb.avgpool(sx)
    y = pb.scale_add(sx, external(pb, gate, precision), external(pb, skip, precision))
    plan = pb.build(); plan.bind(torch.zeros(1, device=DEV), {})
    plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
    check_op(nchw(plan.tensor(pooled)), x.mean(dim=(2, 3), keepdim=True), precision)
    check_op(nchw(plan.tensor(y)), x * gate + skip, precision)
    # h-swish / h-sigmoid epilogues of the 1x1 conv (CUDA-core and, in bf16, tensor-core kernels)
    w = torch.randn(32, C, 1, 1, generator=g) * 0.3; b = torch.randn(32, generator=g)
    for act, fn in (("hswish", hswish), ("hsigmoid", hsigmoid)):
        for tc in ((False, True) if precision == "bf16" else (False,)):
            pb = builder(B, precision, tc=tc)
            y = pb.conv([external(pb, x, precision)], w.to(DEV), b.to(DEV), act=act)
            assert bool(pb.ops[-1].flags & 8) == tc
            check_op(run_op(pb, y), fn(F.conv2d(x, w, b)), precision, 2e-2 if tc else None)


@pytest.mark.parametrize("mode", ["fp32", "bf16", "bf16tc"])
def test_conv_reads_channel_slices(mode):
    """cpb200_op.src_pitch: 1x1 convs reading channel slices of ONE wide NHWC tensor (the fused-head layout:
    a single 3x3 conv writes all six hidden maps, each 1x1 head conv reads its slice through the pitch field)."""
    precision = "fp32" if mode == "fp32" else "bf16"
    B, C, H, W, hc = 2, 32, 16, 24, 64
    g = torch.Generator().manual_seed(6)
    x = torch.randn(B, C, H, W, generator=g).bfloat16().float()
    w3 = (torch.randn(3 * hc, C, 3, 3, generator=g) * 0.1).bfloat16().float(); b3 = torch.randn(3 * hc, generator=g)
    hid_ref = F.relu(F.conv2d(x, w3, b3, padding=1))
    pb = builder(B, precision, tc=(mode == "bf16tc"))
    hid = pb.conv([external(pb, x, precision)], w3.to(DEV), b3.to(DEV), stride=1, pad=1, relu=True)
    outs, refs = {}, []
    for i, co in enumerate((5, 34, 17)):
        w1 = (torch.randn(co, hc, 1, 1, generator=g) * 0.2).bfloat16().float(); b1 = torch.randn(co, generator=g)
        sl = pb.channel_slice(hid, i * hc, hc)
        dst = pb.output(co, H, W, f"o{i}")
        pb.conv([sl], w1.to(DEV), b1.to(DEV), out="nchw", dst=dst)
        assert pb.ops[-1].srcs[0].pitch == 3 * hc
        outs[f"o{i}"] = torch.zeros(B, co, H, W, device=DEV)
        hr = hid_ref[:, i * hc:(i + 1) * hc]
        refs.append(F.conv2d(hr if precision == "fp32" else hr.bfloat16().float(), w1, b1))
    plan = pb.build(); plan.bind(torch.zeros(1, device=DEV), outs)
    plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
    for i, ref in enumerate(refs):
        check_op(outs[f"o{i}"].cpu(), ref, precision, 2e-2 if precision == "bf16" else None)

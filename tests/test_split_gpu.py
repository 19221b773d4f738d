"""GPU parity tests of the split-operand precisions ('fp16x2', 'bf16x2': every value carried as hi + lo 16-bit planes,
products evaluated as hi*hi + hi*lo + lo*hi on wgmma with fp32 accumulation) — the tensor-core path that is meant to
reproduce the reference's fp32 arithmetic (lib/models/model.py:57-59 runs cuDNN fp32 convs and the fp32-only DCNv2,
DCNv2/src/cuda/dcn_v2_cuda.cu:58).

Tolerances (floating point, written here as the task requires), against a float64 evaluation of the same op:
  fp16x2, one op    : |err| <= 1e-5 * max|ref|   (operands 2^-22, dropped lo*lo 2^-22, fp32 accumulation, output re-split)
  bf16x2, one op    : |err| <= 3e-4 * max|ref|   (operands / dropped term 2^-16..2^-17)
  fp16x2, network   : the SAME bound the fp32 CUDA-core path is held to: |err| <= 5e-4 max|ref|, relative L2 <= 2e-4
                      against the reference-generated goldens (expected: ~5e-6 relative L2)
  bf16x2, network   : relative L2 <= 5e-4
  decoded rows      : matched on bbox + score, then element-wise 1e-3 * max(1, |ref|)   (north-star tolerance)
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"
OP_TOL = {"fp16x2": 1e-5, "bf16x2": 3e-4}
PRECS = ["fp16x2", "bf16x2"]


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().to(DEV, torch.float32)


def _nchw(t):
    return t.double().permute(0, 3, 1, 2).contiguous().cpu()


def _builder(B, precision):
    from centerpose_b200.plan import PlanBuilder
    return PlanBuilder(B, 1, 1, precision, torch.device(DEV))


def _run(pb, y):
    plan = pb.build()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return plan.tensor(y).clone()


def _close(got, ref, precision, what=""):
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-30
    assert err <= OP_TOL[precision] * scale, (what, precision, err, scale, err / scale)


SPLIT_CASES = [
    # cins, cout, k, stride, H, W, res, relu, out
    ([64], 64, 3, 1, 16, 16, False, True, "act"),        # halo kernel, resident weights, N-concatenated MMA
    ([64], 64, 3, 1, 40, 48, True, True, "act"),         # partial tiles, residual
    ([128], 128, 3, 1, 24, 16, True, True, "act"),       # halo kernel, streamed [hi|lo] weight stages, two K slabs
    ([64], 256, 3, 1, 32, 32, False, True, "act"),       # head 3x3: BN = 256 -> three N = 256 MMAs
    ([256], 512, 3, 1, 16, 16, True, True, "act"),       # two N tiles
    ([128], 27, 3, 1, 24, 24, False, False, "f32"),      # DCN offset/mask conv: fp32 out, cout 27
    ([16], 16, 3, 1, 64, 64, False, True, "act"),        # SIMT-fed kernel C=16 s1
    ([16], 32, 3, 2, 37, 51, False, True, "act"),        # C=16 s2, partial tiles
    ([32], 64, 3, 2, 50, 30, False, True, "act"),        # C=32 s2 (plane-granular ring of 3 stages)
    ([32], 32, 3, 1, 40, 24, True, True, "act"),         # C=32 s1 + residual
    ([32], 64, 1, 1, 16, 24, False, False, "act"),       # tap-per-stage kernel: 1x1, BK=32
    ([128], 256, 3, 2, 32, 32, False, True, "act"),      # stride 2, BN=256 (two stages of 96 KB)
    ([64], 128, 3, 2, 32, 48, False, True, "act"),       # stride 2, N-concatenated
    ([128, 128, 64, 128], 128, 1, 1, 16, 16, False, True, "act"),   # Root: 4 K-slab inputs
    ([512, 512, 256], 512, 1, 1, 8, 8, False, True, "act"),         # TW=8 tiles
    ([256], 34, 1, 1, 32, 32, False, False, "nchw"),     # head 1x1 -> NCHW fp32 logits (hps)
    ([256], 1, 1, 1, 24, 40, False, False, "nchw"),      # head 1x1 (hm), partial tiles
    ([512], 512, 3, 1, 4, 4, True, True, "act"),         # map narrower than 8 pixels: fp32 island (CONVERT, SIMT conv, CONVERT)
]


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("cins,cout,k,stride,H,W,res,relu,out", SPLIT_CASES)
def test_conv_split(precision, cins, cout, k, stride, H, W, res, relu, out):
    B = 3
    g = torch.Generator().manual_seed(sum(cins) * 7 + cout + k + stride)
    xs = [torch.randn(B, c, H, W, generator=g) for c in cins]
    w = torch.randn(cout, sum(cins), k, k, generator=g) / (sum(cins) * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    pad = k // 2
    ref = F.conv2d(torch.cat(xs, 1).double(), w.double(), b.double(), stride=stride, padding=pad)
    r = None
    if res:
        r = torch.randn(ref.shape, generator=g)
        ref = ref + r.double()
    if relu:
        ref = F.relu(ref)
    pb = _builder(B, precision)
    sx = [pb.external(_nhwc(x)) for x in xs]
    sr = pb.external(_nhwc(r)) if res else None
    if out == "nchw":
        dst = pb.output(cout + 3, ref.shape[2], ref.shape[3], "o")
        buf = torch.zeros(B, cout + 3, ref.shape[2], ref.shape[3], device=DEV)
        pb.conv(sx, w.to(DEV), b.to(DEV), stride=stride, pad=pad, relu=relu, out="nchw", dst=dst, ch_off=2)
        assert pb.ops[-1].flags & 8
        plan = pb.build(); plan.bind(torch.zeros(1, device=DEV), {"o": buf})
        plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
        assert buf[:, :2].abs().max().item() == 0 and buf[:, cout + 2:].abs().max().item() == 0
        _close(buf[:, 2:cout + 2].double().cpu(), ref, precision, "nchw")
        return
    y = pb.conv(sx, w.to(DEV), b.to(DEV), stride=stride, pad=pad, relu=relu, res=sr, out=out)
    if W // stride >= 8:
        assert any(o.type == 1 and (o.flags & 8) for o in pb.ops), "op was not routed to the tensor-core path"
    else:
        assert [o.type for o in pb.ops].count(11) >= 2, "expected an fp32 island"
    _close(_nchw(_run(pb, y)), ref, precision, "conv")


@pytest.mark.parametrize("precision", PRECS)
def test_split_roundtrip_maxpool_upadd_stem(precision):
    from centerpose_b200.plan import split_planes
    B = 2
    g = torch.Generator().manual_seed(2)
    # CONVERT both ways through an fp32 island op that is the identity on the values: max-pool 1x1
    t = torch.randn(B, 32, 16, 20, generator=g) * 3
    for (k, s, p) in ((2, 2, 0), (3, 2, 1)):
        pb = _builder(B, precision)
        y = pb.maxpool(pb.external(_nhwc(t)), k, s, p)
        # exact on the values the planes represent
        tq = split_planes(t, pb.torch16).float().sum(0)
        assert torch.equal(_run(pb, y).permute(0, 3, 1, 2).cpu(), F.max_pool2d(tq, k, s, p))
    # depthwise deconv (f = 2 and f = 4) + skip
    for f in (2, 4):
        C = 32
        xx = torch.randn(B, C, 6, 7, generator=g)
        ww = torch.rand(C, 1, 2 * f, 2 * f, generator=g)
        ref_up = F.conv_transpose2d(xx.double(), ww.double(), None, stride=f, padding=f // 2, groups=C)
        skip = torch.randn(ref_up.shape, generator=g)
        pb = _builder(B, precision)
        y = pb.up_add(pb.external(_nhwc(xx)), pb.external(_nhwc(skip)), ww.to(DEV))
        _close(_nchw(_run(pb, y)), ref_up + skip.double(), precision, "up_add")
    # stems: stride 1 on the tensor cores (16 and 64 channels, partial tiles); stride 2 (ResNet 7x7, HRNet 3x3) as
    # space-to-depth (OP_S2D) + a stride-1 5x5 / 3x3 conv over 16 channels on the tensor cores; odd sizes and
    # CPB200_S2D_STEM=0 through the fp32 island
    for (co, k, stride, H, W, s2d) in ((16, 7, 1, 48, 40, None), (16, 7, 1, 21, 37, None), (64, 7, 1, 16, 24, None),
                                       (64, 7, 2, 38, 50, True), (64, 3, 2, 64, 48, True), (64, 7, 2, 64, 32, True),
                                       (64, 7, 2, 37, 50, False), (64, 7, 2, 38, 50, "off")):
        x = torch.randn(B, 3, H, W, generator=g)
        w = torch.randn(co, 3, k, k, generator=g) * 0.1; b = torch.randn(co, generator=g)
        ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=k // 2))
        pb = _builder(B, precision); pb.H, pb.W = H, W
        if s2d == "off":
            os.environ["CPB200_S2D_STEM"] = "0"
        try:
            y = pb.stem(pb.input(3), w.to(DEV), b.to(DEV), k, stride, k // 2, relu=True)
        finally:
            os.environ.pop("CPB200_S2D_STEM", None)
        if stride == 1:
            assert pb.ops[0].flags & 8
        elif s2d is True:
            assert [o.type for o in pb.ops] == [12, 1] and pb.ops[1].flags & 8 and pb.ops[1].k == ((k + 1) // 2 + 1,) * 2
        else:
            assert pb.ops[0].type == 2 and not (pb.ops[0].flags & 8)
        plan = pb.build(); plan.bind(x.to(DEV), {}); plan.run(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        _close(_nchw(plan.tensor(y)), ref, precision, f"stem{co}k{k}s{stride}")


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("ci,co,H,W,gain", [(64, 64, 16, 16, 1.5), (128, 64, 24, 40, 1.5), (256, 256, 16, 16, 0.3), (512, 256, 8, 8, 0.3),
                                            (64, 128, 33, 20, 1.5)])
def test_dcn_split(precision, ci, co, H, W, gain):
    """wgmma DCN on split operands (both planes gathered, fp32 blend, sample re-split) vs the float64 oracle.  Offsets
    with gain 1.5 put many samples out of bounds.  The sampling positions come from the split-precision offset conv, so
    the comparison includes its error: tolerance 4x the single-op bound."""
    from oracle import dcn_ref
    B = 2
    g = torch.Generator().manual_seed(ci * 3 + co)
    x = torch.randn(B, ci, H, W, generator=g)
    w = torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5; b = torch.randn(co, generator=g)
    ow = torch.randn(27, ci, 3, 3, generator=g) * (gain / (ci * 9) ** 0.5); ob = torch.randn(27, generator=g)
    ref = F.relu(dcn_ref.dcn_module_forward(x.double(), w.double(), b.double(), ow.double(), ob.double()))
    pb = _builder(B, precision)
    y = pb.dcn(pb.external(_nhwc(x)), w.to(DEV), b.to(DEV), ow.to(DEV), ob.to(DEV), relu=True)
    assert pb.ops[-1].type == 5 and pb.ops[-1].flags & 8, "DCN op was not routed to the tensor-core path"
    got = _nchw(_run(pb, y))
    err = (got - ref).abs().max().item(); scale = ref.abs().max().item()
    # a sample whose fractional position sits within rounding of an integer boundary flips corners: bound the bulk by
    # relative L2 and the outliers loosely
    rel = ((got - ref).norm() / ref.norm()).item()
    assert rel <= 4 * OP_TOL[precision] and err <= 40 * OP_TOL[precision] * scale, (precision, rel, err, scale)


def test_dcn_split_zero_offset_identity():
    """DCNv2/test.py:31-66 on the split wgmma DCN: zero offsets, mask 0.5, identity weights => 2*out == in, up to the
    accumulator-bias compensation factor 1 + beta * 36 = 1 + 6e-7 the host folds into acc_scale (plan.rz_compensation);
    exact with CPB200_RZ_COMP=0 (checked too)."""
    B, C, H, W = 2, 64, 24, 16
    x = torch.randint(-8, 9, (B, C, H, W), generator=torch.Generator().manual_seed(0)).float()
    w = torch.zeros(C, C, 3, 3)
    for c in range(C):
        w[c, c, 1, 1] = 1.0
    for precision in PRECS:
        pb = _builder(B, precision)
        y = pb.dcn(pb.external(_nhwc(x)), w.to(DEV), torch.zeros(C, device=DEV),
                   torch.zeros(27, C, 3, 3, device=DEV), torch.zeros(27, device=DEV), relu=False)
        assert pb.ops[-1].flags & 8
        out = _run(pb, y).permute(0, 3, 1, 2).cpu()
        assert (2 * out - x).abs().max().item() <= 1e-6 * 8, precision
        os.environ["CPB200_RZ_COMP"] = "0"
        try:
            pb = _builder(B, precision)
            y = pb.dcn(pb.external(_nhwc(x)), w.to(DEV), torch.zeros(C, device=DEV),
                       torch.zeros(27, C, 3, 3, device=DEV), torch.zeros(27, device=DEV), relu=False)
            out = _run(pb, y).permute(0, 3, 1, 2).cpu()
        finally:
            os.environ.pop("CPB200_RZ_COMP", None)
        assert torch.equal(2 * out, x), precision


def _model(precision, arch="dla_34"):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg(arch)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    sd = conditioned_state_dict(m.state_dict(), 317)
    m.load_state_dict(sd)
    return m.to(DEV).set_precision(precision), sd


def _net_err(got, ref):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    return np.abs(got - ref).max() / np.abs(ref).max(), np.linalg.norm(got - ref) / np.linalg.norm(ref)


NET_TOL = {"fp16x2": (5e-4, 2e-4), "bf16x2": (2e-3, 5e-4)}


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("arch,tag", [("dla_34", "dla34_128"), ("dla_34", "dla34_96x160"), ("res_50", "res50_128"),
                                      ("hrnet", "hrnet32_128"), ("hrnet", "hrnet32_256x320"), ("mobilenetv3", "mbv3_128x160")])
def test_network_split_matches_reference_golden(precision, arch, tag):
    """Whole network on split operands against the reference's own head maps (goldens generated by running the
    unmodified reference, oracle/make_golden.py).  Small inputs also exercise the fp32 islands (maps < 8 pixels wide,
    HRNet's upsample-add, MobileNetV3's depthwise / SE ops, the stride-2 stem)."""
    from oracle.init_recipe import synth_images
    g = np.load(os.path.join(GOLD, tag + ".npz"))
    B, H, W = [int(v) for v in g["shape"]]
    st = int(g["stride"]) if "stride" in g.files else 1
    m, _ = _model(precision, arch)
    maps = torch.cat(m(synth_images(B, H, W, 317).to(DEV)), dim=1).cpu().numpy()[:, :, ::st, ::st]
    assert maps.shape == g["maps"].shape
    mx, rel = _net_err(maps, g["maps"])
    print(f"{arch} {tag} {precision}: max/max {mx:.3e} relL2 {rel:.3e}")
    assert mx <= NET_TOL[precision][0] and rel <= NET_TOL[precision][1], (mx, rel)


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("arch,tag", [("dla_34", "dla34_512"), ("res_50", "res50_512"), ("hrnet", "hrnet32_512"), ("mobilenetv3", "mbv3_512")])
def test_network_split_512_end_to_end(precision, arch, tag):
    """BASELINE.json's 512x512 configuration: head maps AND decoded detections of the split tensor-core path against the
    reference's own outputs (experiments/*_512x512.yaml:31-36).  Rows are matched on bbox + score (top-K is
    discontinuous), then compared element-wise at the north-star tolerance 1e-3."""
    from centerpose_b200 import multi_pose_decode
    from oracle.init_recipe import synth_images
    from tests.util import match_rows
    g = np.load(os.path.join(GOLD, tag + ".npz"))
    B, H, W = [int(v) for v in g["shape"]]
    st = int(g["stride"]) if "stride" in g.files else 1
    m, _ = _model(precision, arch)
    outs = m(synth_images(B, H, W, 317).to(DEV))
    maps = torch.cat(outs, dim=1).cpu().numpy()[:, :, ::st, ::st]
    mx, rel = _net_err(maps, g["maps"])
    hm, wh, hps, reg, hm_hp, hp_off = outs
    dets = multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_off, K=100, apply_sigmoid=True).cpu().numpy()
    rows, elems = match_rows(dets[0], g["dets"][0], tol=1e-3, box_tol=2e-2)
    print(f"{arch} 512 {precision}: max/max {mx:.3e} relL2 {rel:.3e} rows matched {rows:.3f} elements within 1e-3 {elems:.4f}")
    assert mx <= NET_TOL[precision][0] and rel <= NET_TOL[precision][1], (mx, rel)
    if precision == "fp16x2":
        assert rows >= 0.99 and elems >= 0.99, (rows, elems)
    else:
        assert rows >= 0.9 and elems >= 0.95, (rows, elems)


@pytest.mark.parametrize("precision", PRECS)
def test_elementwise_ops_on_planes(precision):
    """CPB200_OP_DWCONV / AVGPOOL / SCALE_ADD / UPSAMPLE_ADD take split planes directly (no fp32 island: the program holds
    no CONVERT): fp32 arithmetic on hi + lo, result re-split   (mobilenetv3.py:84-147, pose_higher_hrnet.py:186-232)."""
    from centerpose_b200.plan import OP_CONVERT
    from oracle.mobilenet_ref import hswish
    g = torch.Generator().manual_seed(23)
    B, C, H, W = 2, 48, 13, 18
    x = torch.randn(B, C, H, W, generator=g) * 2
    for k, stride, act, fn in ((3, 1, "relu", F.relu), (5, 2, "hswish", hswish), (5, 1, None, lambda t: t), (3, 2, "hswish", hswish),
                                (7, 1, "relu", F.relu)):
        w = torch.randn(C, 1, k, k, generator=g) * 0.3; b = torch.randn(C, generator=g)
        pb = _builder(B, precision)
        y = pb.dwconv(pb.external(_nhwc(x)), w.to(DEV), b.to(DEV), stride=stride, act=act)
        assert [o.type for o in pb.ops] == [8] and pb.ops[0].dtype == pb.act_dtype
        _close(_nchw(_run(pb, y)), fn(F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=k // 2, groups=C)), precision, f"dwconv k{k} s{stride}")
    gate = torch.rand(B, C, 1, 1, generator=g); skip = torch.randn(B, C, H, W, generator=g)
    for with_skip in (True, False):
        pb = _builder(B, precision)
        sx = pb.external(_nhwc(x))
        pooled = pb.keep_result(pb._to_f32(pb.avgpool(sx)))                 # planes in, fp32 (B,1,1,C) out
        y = pb.scale_add(sx, pb.external(_nhwc(gate)), pb.external(_nhwc(skip)) if with_skip else None)
        plan = pb.build(); plan.run(torch.cuda.current_stream().cuda_stream); torch.cuda.synchronize()
        assert sum(o.type == OP_CONVERT for o in plan.pb.ops) == 1    # only the externally supplied gate is converted to fp32
        _close(_nchw(plan.tensor(pooled)), x.double().mean(dim=(2, 3), keepdim=True), precision, "avgpool")
        _close(_nchw(plan.tensor(y)), x.double() * gate.double() + (skip.double() if with_skip else 0), precision, "scale_add")
    for f, relu, with_skip in ((2, True, True), (4, False, True), (8, True, False)):
        xt = torch.randn(B, 32, 5, 7, generator=g); st = torch.randn(B, 32, 5 * f, 7 * f, generator=g)
        pb = _builder(B, precision)
        y = pb.upsample_add(pb.external(_nhwc(xt)), pb.external(_nhwc(st)) if with_skip else None, f, relu=relu)
        assert [o.type for o in pb.ops] == [7]
        ref = F.interpolate(xt.double(), scale_factor=f, mode="nearest") + (st.double() if with_skip else 0)
        _close(_nchw(_run(pb, y)), F.relu(ref) if relu else ref, precision, f"upsample_add x{f}")


def test_split_batch_consistency_and_rebinding():
    """Image i of a batch == the same image alone (bit for bit), and a second forward on the same plan with the first
    call's outputs still held returns independent, correct tensors (outputs are re-bound per call)."""
    from oracle.init_recipe import synth_images
    m, _ = _model("fp16x2")
    x = synth_images(3, 128, 160, seed=9).to(DEV)
    o_all = [t.clone() for t in m(x)]
    o_again = m(x)                                  # same plan, new output tensors, earlier outputs alive
    for a, b in zip(o_all, o_again):
        assert torch.equal(a, b)
    for i in range(3):
        o_i = m(x[i:i + 1])
        for a, b in zip(o_all, o_i):
            assert torch.equal(a[i:i + 1], b), i


@pytest.mark.parametrize("precision", ["bf16", "fp16x2", "bf16x2"])
@pytest.mark.parametrize("B,ci,co,H,W,res", [(5, 64, 256, 64, 64, False),      # head conv shape: two N tiles, streamed weights
                                              (11, 128, 128, 48, 40, True),     # 165 pixel tiles, partial tiles
                                              (10, 256, 256, 32, 32, True)])    # four K slabs
def test_conv_streamed_weights_path(precision, B, ci, co, H, W, res):
    """3x3 convs whose filter bank does not stay resident in shared memory (csrc/net_tc3.cu streams it through a weight
    ring): several N tiles, several K slabs, partial tiles, more pixel tiles than SMs."""
    g = torch.Generator().manual_seed(B * 7 + ci + co)
    x = torch.randn(B, ci, H, W, generator=g)
    w = torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5
    b = torch.randn(co, generator=g)
    r = torch.randn(B, co, H, W, generator=g) if res else None
    if precision == "bf16":
        x = x.bfloat16().float(); w = w.bfloat16().float()
        r = r.bfloat16().float() if res else None
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    if res:
        ref = ref + r.double()
    ref = F.relu(ref)
    from centerpose_b200.plan import PlanBuilder
    pb = PlanBuilder(B, 1, 1, precision, torch.device(DEV))
    if precision == "bf16":
        sx = pb.external(x.permute(0, 2, 3, 1).contiguous().to(DEV, torch.bfloat16))
        sr = pb.external(r.permute(0, 2, 3, 1).contiguous().to(DEV, torch.bfloat16)) if res else None
    else:
        sx = pb.external(_nhwc(x)); sr = pb.external(_nhwc(r)) if res else None
    y = pb.conv([sx], w.to(DEV), b.to(DEV), stride=1, pad=1, relu=True, res=sr)
    got = _nchw(_run(pb, y))
    err = (got - ref).abs().max().item(); scale = ref.abs().max().item()
    tol = 1e-2 if precision == "bf16" else OP_TOL[precision]
    assert err <= tol * scale, (precision, err, scale, err / scale)


@pytest.mark.parametrize("precision", ["fp16x2", "bf16"])
def test_halo_conv_output_rebinding(precision):
    """`dst` of a prepared halo conv is read live (include/centerpose_b200.h, cpb200_prepare_ops): re-binding it after the
    first run must write the new buffer and leave the old one untouched, and a freshly prepared plan must give the same
    bits."""
    from centerpose_b200.plan import PlanBuilder
    g = torch.Generator().manual_seed(77)
    B, ci, co, H, W = 2, 64, 128, 24, 40                     # partial tiles in both directions
    x = torch.randn(B, ci, H, W, generator=g)
    w = torch.randn(co, ci, 3, 3, generator=g) / (ci * 9) ** 0.5
    b = torch.randn(co, generator=g)
    if precision == "bf16":
        x = x.bfloat16().float(); w = w.bfloat16().float()

    def build():
        pb = PlanBuilder(B, 1, 1, precision, torch.device(DEV))
        sx = pb.external(x.permute(0, 2, 3, 1).contiguous().to(DEV, torch.bfloat16)) if precision == "bf16" else pb.external(_nhwc(x))
        y = pb.conv([sx], w.to(DEV), b.to(DEV), stride=1, pad=1, relu=True)
        return pb, y, pb.build()

    st = torch.cuda.current_stream().cuda_stream
    pb, y, plan = build()
    plan.run(st); torch.cuda.synchronize()
    first = plan.tensor(y).clone()
    raw_first = y.buf.clone()
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1))
    err = (_nchw(first) - ref).abs().max().item()
    assert err <= (1e-2 if precision == "bf16" else OP_TOL[precision]) * ref.abs().max().item()
    # re-bind: a fresh, poisoned buffer of the same size
    new = torch.full_like(y.buf, 0x7F)
    y.buf.fill_(0x55)
    i = [k for k in range(plan.n) if plan.pb.ops[k].dst is y][0]
    plan.ops[i].dst = new.data_ptr()
    plan.run(st); torch.cuda.synchronize()
    assert bool((y.buf == 0x55).all()), "the old output buffer was written after re-binding"
    n_used = raw_first.numel() if precision != "bf16" else B * H * W * co * 2
    assert torch.equal(new[:n_used], raw_first[:n_used])
    # a second, independently prepared plan gives the same bits
    pb2, y2, plan2 = build()
    plan2.run(st); torch.cuda.synchronize()
    assert torch.equal(y2.buf[:n_used], raw_first[:n_used])

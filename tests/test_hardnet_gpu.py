"""GPU tests of the HarDNet backbone (centerpose_b200/archs/hardnet.py) and its two element-wise ops,
CPB200_OP_AVGPOOL2 and CPB200_OP_RESIZE_BILINEAR.

Tolerances (against a float64 torch evaluation for the ops, the reference-generated goldens for the network):
  fp32 op        : |err| <= 2e-4 * max|ref|
  bf16 op        : relative L2 <= 1e-2 (inputs already bf16-representable; one output rounding)
  fp16x2 op      : |err| <= 1e-5 * max|ref|;  bf16x2 op: |err| <= 3e-4 * max|ref|
  fp32 network   : |err| <= 5e-4 * max|ref| and relative L2 <= 2e-4 (tests/test_net_gpu.py::_net_close)
  fp16x2 network : the same bound; at 512x512 every reference detection row matched and >= 99.9 % of the values
                   within 1e-3 * max(1, |ref|) (tests/test_split_gpu.py holds DLA-34 to >= 99 %; the two values that
                   move sit on a near-tie of the decode, see the test)
  bf16 network   : relative L2 <= 4e-2 (reported)
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"
PRECS = ["fp32", "bf16", "bf16x2", "fp16x2"]
SPLIT_TOL = {"fp16x2": 1e-5, "bf16x2": 3e-4}

POOL_IN = [(13, 18), (3, 5), (6, 10), (16, 16), (24, 40), (12, 20), (2, 2)]
RESIZE = [((13, 18), (6, 9)), ((1, 2), (3, 5)), ((3, 5), (6, 10)), ((8, 8), (16, 16)), ((12, 20), (24, 40)),
          ((12, 20), (12, 20)), ((2, 3), (1, 1))]


def _builder(B, precision):
    from centerpose_b200.plan import PlanBuilder
    return PlanBuilder(B, 1, 1, precision, torch.device(DEV))


def _external(pb, x, precision):
    """NCHW fp32 -> program input in the precision's storage (split precisions: fp32 in, planes made by the builder)."""
    t = x.permute(0, 2, 3, 1).contiguous()
    return pb.external(t.to(DEV, torch.bfloat16 if precision == "bf16" else torch.float32))


def _run_one(pb, y):
    plan = pb.build()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return plan.tensor(y).double().permute(0, 3, 1, 2).cpu()


def _check(got, ref, precision, what):
    scale = ref.abs().max().item() + 1e-30
    if precision == "fp32":
        assert (got - ref).abs().max().item() <= 2e-4 * scale, what
    elif precision == "bf16":
        rel = ((got - ref).norm() / (ref.norm() + 1e-30)).item()
        assert rel <= 1e-2, (what, rel)
    else:
        err = (got - ref).abs().max().item()
        assert err <= SPLIT_TOL[precision] * scale, (what, err / scale)


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
        pb = _builder(B, precision)
        y = pb.avgpool2(_external(pb, x, precision))
        assert [o.type for o in pb.ops] == [OP_AVGPOOL2] and (y.H, y.W) == (H // 2, W // 2)
        _check(_run_one(pb, y), F.avg_pool2d(x.double(), 2, 2), precision, (H, W))


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("C", [16, 48, 320])
def test_resize_bilinear_op_matches_torch(precision, C):
    """bilinear resize, align_corners=True, to arbitrary sizes (up, down, same size, from a 1-pixel-high map, to 1x1)."""
    from centerpose_b200.plan import OP_RESIZE_BILINEAR
    B = 2
    for i, ((H, W), (Ho, Wo)) in enumerate(RESIZE):
        x = _input(B, C, H, W, 200 * C + i, precision)
        pb = _builder(B, precision)
        y = pb.resize_bilinear(_external(pb, x, precision), Ho, Wo)
        assert [o.type for o in pb.ops] == [OP_RESIZE_BILINEAR]
        ref = F.interpolate(x.double(), size=(Ho, Wo), mode="bilinear", align_corners=True)
        _check(_run_one(pb, y), ref, precision, ((H, W), (Ho, Wo)))
    if precision == "fp32":                 # fp32: PyTorch's own fp32 arithmetic, to within a couple of ulps
        x = _input(B, C, 12, 20, 7, precision)
        pb = _builder(B, precision)
        y = pb.resize_bilinear(_external(pb, x, precision), 24, 40)
        ref = F.interpolate(x, size=(24, 40), mode="bilinear", align_corners=True).double()
        assert (_run_one(pb, y) - ref).abs().max().item() <= 4 * 2.0 ** -23 * ref.abs().max().item()


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
        pb = _builder(B, precision)
        pb.avgpool2(_external(pb, x, precision))
        return pb

    def resize():
        pb = _builder(B, precision)
        pb.resize_bilinear(_external(pb, x, precision), 9, 11)
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


def _model(precision):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg("hardnet")
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    sd = conditioned_state_dict(m.state_dict(), 317)
    m.load_state_dict(sd)
    return m.to(DEV).set_precision(precision), sd


def _net_err(got, ref):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    return np.abs(got - ref).max() / np.abs(ref).max(), np.linalg.norm(got - ref) / np.linalg.norm(ref)


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
@pytest.mark.parametrize("tag", ["128", "96x160", "512"])
def test_hardnet_matches_reference_golden(precision, tag):
    """Whole network against the unmodified reference's head maps.  128x128 reaches a 2x2 deepest map, 96x160 odd pools
    and a resize from a 1-pixel-high map (fp16x2: the narrow maps run in fp32 islands); at 512x512 the decoded rows
    are compared too."""
    from centerpose_b200 import multi_pose_decode
    from oracle.init_recipe import synth_images
    from tests.util import match_rows
    g = np.load(os.path.join(GOLD, f"hardnet_{tag}.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    st = int(g["stride"])
    m, _ = _model(precision)
    outs = m(synth_images(B, H, W, 317).to(DEV))
    maps = torch.cat(outs, dim=1).cpu().numpy()[:, :, ::st, ::st]
    assert maps.shape == g["maps"].shape
    mx, rel = _net_err(maps, g["maps"])
    print(f"hardnet {tag} {precision}: max/max {mx:.3e} relL2 {rel:.3e}")
    assert mx <= 5e-4 and rel <= 2e-4, (mx, rel)
    if tag != "512":
        return
    dets = multi_pose_decode(outs[0], outs[1], outs[2], reg=outs[3], hm_hp=outs[4], hp_offset=outs[5], K=100,
                             apply_sigmoid=True).cpu().numpy()
    rows, elems = match_rows(dets[0], g["dets"][0], tol=1e-3, box_tol=2e-2)
    print(f"hardnet 512 {precision}: rows matched {rows:.3f}, elements within 1e-3 {elems:.4f}")
    if precision == "fp32":
        assert rows >= 0.9 and elems >= 0.97, (rows, elems)
    else:
        # All 100 rows match.  Values: >= 99.9 %, not 100 %.  Keypoint 1 of reference row 98 sits on a near-tie of the
        # decode's keypoint-heat-map snapping.  Perturbing the reference's exact head maps by 2e-6 relative noise moves
        # that keypoint to the other candidate in 3 of 5 seeds.  The fp32 CUDA-core path (maps 3e-7 from the reference)
        # and fp16x2 (1.5e-6) both land on the other candidate: 2 of 5 600 values.
        assert rows == 1.0 and elems >= 0.999, (rows, elems)
        from centerpose_b200.plan import OP_CONVERT
        plan = next(iter(m._plans.values()))
        assert sum(o.type == OP_CONVERT for o in plan.ops) == 0     # no fp32 island at 512x512


def test_hardnet_512_bf16_reported():
    from oracle.init_recipe import synth_images
    g = np.load(os.path.join(GOLD, "hardnet_512.npz"))
    m, _ = _model("bf16")
    maps = torch.cat(m(synth_images(1, 512, 512, 317).to(DEV)), dim=1).cpu().numpy()[:, :, ::4, ::4]
    mx, rel = _net_err(maps, g["maps"])
    print(f"hardnet 512 bf16: max/max {mx:.3e} relL2 {rel:.3e}")
    assert rel <= 4e-2, rel


def test_hardnet_batch_consistency_and_output_rebinding():
    """Image i of a 64-image batch equals the same image alone, bit for bit, and a second forward on the same plan while
    the first call's outputs are alive returns independent, correct tensors (tests/test_net_gpu.py pattern)."""
    from oracle.init_recipe import synth_images
    B = 64
    m, _ = _model("bf16")
    x1 = synth_images(B, 128, 160, seed=21).to(DEV)
    x2 = synth_images(B, 128, 160, seed=22).to(DEV)
    ref1 = [t.clone() for t in m(x1)]
    m.invalidate()
    ref2 = [t.clone() for t in m(x2)]
    m.invalidate()
    o1 = m(x1)
    o2 = m(x2)
    o3 = m(x1)
    for a, b in zip(o1, ref1):
        assert torch.equal(a, b)
    for a, b in zip(o2, ref2):
        assert torch.equal(a, b)
    for a, b in zip(o3, ref1):
        assert torch.equal(a, b)
    assert len({t.data_ptr() for t in o1 + o2 + o3}) == 18
    for i in (0, B // 2, B - 1):
        alone = m(x1[i:i + 1])
        for a, b in zip(ref1, alone):
            assert torch.equal(a[i:i + 1], b), i


def test_hardnet_detector_run_batch_fused():
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle import post_process_ref
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg("hardnet")
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    x = torch.randn(2, 3, 512, 512, generator=torch.Generator().manual_seed(1))
    out = det.run_batch_fused(x, [post_process_ref.make_meta(480, 640), post_process_ref.make_meta(512, 512)])
    assert out.shape == (2, 100, 56) and np.isfinite(out).all()
    assert (out[:, :, 4] > 0).all()

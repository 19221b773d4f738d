"""GPU tests of the MobileNetV2 and GhostNet backbones (centerpose_b200/archs/mobilenetv2.py, archs/ghostnet.py) and of
the device work they added: the ReLU6 / clip01 epilogue activations (CPB200_FLAG_RELU6 / CPB200_FLAG_CLIP01), the bias
form of CPB200_OP_DWDECONV_ADD (k 2 / stride 2 deconv + folded BN + ReLU + skip) and the 4x bilinear upscale.

Tolerances:
  ops, "int" data : exact, element by element (tests/replay.py: integers that every format holds exactly)
  ops, randn data : fp32 |err| <= 2e-4 max|ref|; bf16 relative L2 <= 1e-2; fp16x2 |err| <= 1e-5 max|ref|;
                    bf16x2 |err| <= 3e-4 max|ref|   (tests/test_hardnet_gpu.py)
  fp32 / fp16x2 network : |err| <= 5e-4 max|ref| and relative L2 <= 2e-4 (tests/test_hardnet_gpu.py)
  bf16x2 network  : |err| <= 5e-3 max|ref| and relative L2 <= 2e-3 (16 significand bits per plane)
  bf16 network    : relative L2 <= 4e-2 (GhostNet: 1.1e-2 measured); MobileNetV2 <= 1.5e-1 (7.6e-2 at 96x160, 1.0e-1 at
                    512x512 measured on an H100: plain bf16 activations through 52 narrow layers; bf16 is the fast
                    mode, with no parity claim)
  decode at 512x512: fp16x2 every reference row matched and every value within 1e-3 * max(1, |ref|) (the project's
                    headline criterion); fp32 (CUDA-core summation order) >= 90 % rows, >= 97 % values, as for HarDNet.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.kernel_routes import CASES
from tests.layer_census import Record
from tests.replay import _data, _reference, _replay

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"
PRECS = ["fp32", "bf16", "bf16x2", "fp16x2"]
SPLIT_TOL = {"fp16x2": 1e-5, "bf16x2": 3e-4}


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
def _builder(B, precision):
    from centerpose_b200.plan import PlanBuilder
    return PlanBuilder(B, 1, 1, precision, torch.device(DEV))


def _external(pb, x, precision):
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
            pb = _builder(B, precision)
            y = pb.up_add(_external(pb, x, precision), _external(pb, skip, precision) if skip_on else None, w, b=b,
                          act="relu", stride=2, pad=0)
            assert [o.type for o in pb.ops] == [OP_DWDECONV_ADD] and (y.H, y.W) == (2 * H, 2 * W)
            ref = F.relu(F.conv_transpose2d(x.double(), w.double(), b.double(), stride=2, groups=C))
            if skip_on:
                ref = ref + skip.double()
            got = _run_one(pb, y)
            if leg == "int":
                assert torch.equal(got, ref), (precision, C, H, W)
            else:
                _check(got, ref, precision, (C, H, W))


def test_dwdeconv_activation_needs_bias():
    """An activation flag on the bias-less form is rejected (CPB200_ERR_ARG) before anything is launched."""
    pb = _builder(1, "fp32")
    x = torch.randn(1, 16, 4, 4)
    pb.up_add(_external(pb, x, "fp32"), None, torch.randn(16, 1, 4, 4))
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
    pb = _builder(B, precision)
    xs = _external(pb, x, precision)
    h = pb.conv([pb.avgpool(xs)], w1, b1, act="relu")
    gate = pb.conv([h], w2, b2, act="clip01")
    y = pb.scale_add(xs, gate)
    s = F.relu(F.conv2d(x.double().mean(dim=(2, 3), keepdim=True), w1.double(), b1.double()))
    gd = F.conv2d(s, w2.double(), b2.double())
    assert (gd < 0).any() and (gd > 1).any()
    ref = x.double() * gd.clamp(0, 1)
    _check(_run_one(pb, y), ref, precision, "se")


@pytest.mark.parametrize("precision", PRECS)
def test_resize_bilinear_4x_upscale(precision):
    """GhostNet's fixed 128 x 128 resize: 2x (512 input), 4x (256 input) and a non-square 4x / 3.2x, in every format."""
    B, C = 1, 80
    for i, (H, W) in enumerate([(64, 64), (32, 32), (32, 40)]):
        x = _rnd(torch.randn(B, C, H, W, generator=torch.Generator().manual_seed(i)) * 3, precision)
        pb = _builder(B, precision)
        y = pb.resize_bilinear(_external(pb, x, precision), 128, 128)
        ref = F.interpolate(x.double(), size=(128, 128), mode="bilinear", align_corners=True)
        _check(_run_one(pb, y), ref, precision, (H, W))


# ------------------------------------------------------------------------------------------- networks
def _model(arch, precision):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg(arch)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    m.load_state_dict(conditioned_state_dict(m.state_dict(), 317))
    return m.to(DEV).set_precision(precision)


def _net_err(got, ref):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    return np.abs(got - ref).max() / np.abs(ref).max(), np.linalg.norm(got - ref) / np.linalg.norm(ref)


NETS = [("mobilenetv2", "mbv2_512"), ("mobilenetv2", "mbv2_96x160"), ("ghostnet", "ghostnet_512")]


@pytest.mark.parametrize("precision", PRECS)
@pytest.mark.parametrize("arch,tag", NETS)
def test_network_matches_reference_golden(arch, tag, precision):
    """Whole network against the unmodified reference's head maps; at 512x512 the decoded rows too."""
    from centerpose_b200 import multi_pose_decode
    from oracle.init_recipe import synth_images
    from tests.util import match_rows
    g = np.load(os.path.join(GOLD, f"{tag}.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    st = int(g["stride"])
    m = _model(arch, precision)
    outs = m(synth_images(B, H, W, 317).to(DEV))
    maps = torch.cat(outs, dim=1).cpu().numpy()[:, :, ::st, ::st]
    assert maps.shape == g["maps"].shape
    mx, rel = _net_err(maps, g["maps"])
    print(f"{tag} {precision}: max/max {mx:.3e} relL2 {rel:.3e}")
    if precision in ("fp32", "fp16x2"):
        assert mx <= 5e-4 and rel <= 2e-4, (mx, rel)
    elif precision == "bf16x2":
        assert mx <= 5e-3 and rel <= 2e-3, (mx, rel)
    else:
        assert rel <= (1.5e-1 if arch == "mobilenetv2" else 4e-2), rel
    if H != 512 or precision not in ("fp32", "fp16x2"):
        return
    dets = multi_pose_decode(outs[0], outs[1], outs[2], reg=outs[3], hm_hp=outs[4], hp_offset=outs[5], K=100,
                             apply_sigmoid=True).cpu().numpy()
    rows, elems = match_rows(dets[0], g["dets"][0], tol=1e-3, box_tol=2e-2)
    print(f"{tag} {precision}: rows matched {rows:.3f}, elements within 1e-3 {elems:.4f}")
    if precision == "fp32":
        assert rows >= 0.9 and elems >= 0.97, (rows, elems)
    else:
        assert rows == 1.0 and elems == 1.0, (rows, elems)


@pytest.mark.parametrize("arch,tag", [("mobilenetv2", "mbv2_512"), ("ghostnet", "ghostnet_512")])
def test_detector_run_batch_fused_matches_reference_rows(arch, tag):
    """run_batch_fused (fp16x2 forward + decode + back-projection on the device) against the reference's decoded rows
    of its own maps, back-projected by the oracle's post-process, for a 512x512 image."""
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle import post_process_ref
    from oracle.init_recipe import conditioned_state_dict, synth_images
    from tests.util import match_rows
    g = np.load(os.path.join(GOLD, f"{tag}.npz"))
    cfg = default_cfg(arch)
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    meta = post_process_ref.make_meta(512, 512)
    out = det.run_batch_fused(synth_images(1, 512, 512, 317), [meta])
    ref = post_process_ref.detector_post_process(g["dets"], meta)[1]
    assert out.shape == (1, 100, 56) and np.isfinite(out).all()
    rows, elems = match_rows(out[0], ref, tol=1e-3, box_tol=8e-2)
    print(f"{tag} run_batch_fused: rows matched {rows:.3f}, elements within 1e-3 {elems:.4f}")
    assert rows == 1.0 and elems == 1.0, (rows, elems)


@pytest.mark.parametrize("arch", ["mobilenetv2", "ghostnet"])
def test_run_images_returns_rows(arch):
    """det.run_images on raw BGR images of two sizes returns detection rows for each (GhostNet: the heads always see
    the 128 x 128 map, as in the reference)."""
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg(arch)
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8), rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)]
    res = det.run_images(imgs)
    assert len(res) == 2
    for r in res:
        r = np.asarray(r)
        assert r.ndim == 2 and r.shape[1] == 56 and len(r) > 0 and np.isfinite(r).all()

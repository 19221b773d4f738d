"""Shared test helpers: the seeded model and the golden comparison of the network tests (tests/test_backbones_gpu.py),
the plan builder, I/O and per-precision bound of the op tests, and the tie-/discontinuity-aware comparison of decoded
detections.  A helper module: it holds no tests."""
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DEV = "cuda:0"

# one op against a float64 (or fp32) torch evaluation: max|err| / max|ref| for fp32 (fp32 accumulation, different
# summation order) and the split precisions (fp16x2: operands 2^-22, dropped lo*lo 2^-22, fp32 accumulation, output
# re-split; bf16x2: operands / dropped term 2^-16..2^-17); relative L2 for bf16 (one output rounding)
OP_TOL = {"fp32": 2e-4, "bf16": 1e-2, "fp16x2": 1e-5, "bf16x2": 3e-4}


# MODEL.EXTRA of experiments/hrnet_w48_512.yaml (HRNet-W48; its INTERMEDIATE_CHANNEL is 48, HEAD_CONV 64 as W32's)
HRNET_W48_EXTRA = {
    "STAGE2": {"NUM_MODULES": 1, "NUM_BRANCHES": 2, "BLOCK": "BASIC", "NUM_BLOCKS": [4, 4], "NUM_CHANNELS": [48, 96]},
    "STAGE3": {"NUM_MODULES": 4, "NUM_BRANCHES": 3, "BLOCK": "BASIC", "NUM_BLOCKS": [4, 4, 4],
               "NUM_CHANNELS": [48, 96, 192]},
    "STAGE4": {"NUM_MODULES": 3, "NUM_BRANCHES": 4, "BLOCK": "BASIC", "NUM_BLOCKS": [4, 4, 4, 4],
               "NUM_CHANNELS": [48, 96, 192, 384]},
}

# The eight configurations the network tests run: the seven archs' defaults and HRNet-W48 ("hrnet_w48").
ARCHS = ["dla_34", "res_50", "hrnet", "hrnet_w48", "mobilenetv3", "hardnet", "mobilenetv2", "ghostnet"]

# Network inputs the detector builds at deployment (TEST.FIX_RES false pads an image of h x w at a test scale to
# (h | 31) + 1 by (w | 31) + 1): a small image at scale 0.5 (32x32, 64x64), extreme strips (32x640, 640x32: deep maps of
# one pixel), COCO's 640x213 / 213x640 (224x640, 640x224), 427x640 (448x640) and 480x640 at scale 1.5 (736x960).  B = 1.
DEPLOY_SHAPES = [(32, 32), (64, 64), (32, 640), (640, 32), (224, 640), (640, 224), (448, 640), (736, 960)]
# (arch, H, W) the reference cannot run, with the reason; the product refuses them when it builds the plan
_NO_POOL = "HarDNet's %s deepest map has no 2x2 average pool (the reference's AvgPool2d raises)"
TOO_SMALL = {("hardnet", 32, 32): _NO_POOL % "1x1", ("hardnet", 32, 640): _NO_POOL % "1x20",
             ("hardnet", 640, 32): _NO_POOL % "20x1"}


def config(arch):
    """the default config of ``arch``, one of ARCHS ("hrnet_w48": the 'hrnet' arch with HRNET_W48_EXTRA)"""
    from centerpose_b200.config import default_cfg
    if arch != "hrnet_w48":
        return default_cfg(arch)
    cfg = default_cfg("hrnet")
    cfg.MODEL.EXTRA = HRNET_W48_EXTRA
    cfg.MODEL.INTERMEDIATE_CHANNEL = 48
    return cfg


def model(arch, precision, tc=None):
    """``config(arch)`` with the conditioned seed-317 weights (oracle/init_recipe.py), on cuda:0 in ``precision``.
    Returns (model, state_dict)."""
    from centerpose_b200.model import create_model
    from oracle.init_recipe import conditioned_state_dict
    cfg = config(arch)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    sd = conditioned_state_dict(m.state_dict(), 317)
    m.load_state_dict(sd)
    return m.to(DEV).set_precision(precision, tc=tc), sd


def golden_input(tag):
    """``synth_images`` at the shape of tests/golden/<tag>.npz: the input its maps were computed on."""
    from oracle.init_recipe import synth_images
    B, H, W = [int(v) for v in np.load(os.path.join(GOLD, tag + ".npz"))["shape"]]
    return synth_images(B, H, W, 317)


def golden_check(model, tag, outs=None):
    """Run ``model`` on the input of tests/golden/<tag>.npz and compare its head maps, subsampled by the golden's
    ``stride``, with the golden's.  Returns (outputs, max|err| / max|ref|, relative L2, rows); for a golden that holds
    ``dets``, rows is (decoded rows of image 0, the golden's rows of image 0), else None.  ``outs``: compare these
    six head maps (the model's outputs on that input, e.g. one image's slice of a batch) instead of running it."""
    from centerpose_b200 import multi_pose_decode
    g = np.load(os.path.join(GOLD, tag + ".npz"))
    st = int(g["stride"]) if "stride" in g.files else 1
    if outs is None:
        outs = model(golden_input(tag).to(DEV))
    maps = torch.cat(outs, dim=1).cpu().numpy()[:, :, ::st, ::st].astype(np.float64)
    ref = g["maps"].astype(np.float64)
    assert maps.shape == ref.shape, (maps.shape, ref.shape)
    mx = np.abs(maps - ref).max() / np.abs(ref).max()
    rel = np.linalg.norm(maps - ref) / np.linalg.norm(ref)
    rows = None
    if "dets" in g.files:
        hm, wh, hps, reg, hm_hp, hp_off = outs
        dets = multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_off, K=100, apply_sigmoid=True)
        rows = (dets[0].cpu().numpy(), g["dets"][0])
    return outs, mx, rel, rows


def builder(B, precision, tc=None):
    from centerpose_b200.plan import PlanBuilder
    return PlanBuilder(B, 1, 1, precision, torch.device(DEV), tc=tc)


def external(pb, x_nchw, precision):
    """NCHW host tensor -> program input in the precision's storage: bf16 for 'bf16', fp32 otherwise (the split
    precisions take fp32 and the builder makes the planes)."""
    t = x_nchw.permute(0, 2, 3, 1).contiguous()
    return pb.external(t.to(DEV, torch.bfloat16 if precision == "bf16" else torch.float32))


def nchw(t):
    """A device NHWC activation as float64 NCHW on the CPU."""
    return t.double().permute(0, 3, 1, 2).contiguous().cpu()


def run_op(pb, y):
    """Build and run the program, return ``y`` as float64 NCHW on the CPU."""
    plan = pb.build()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return nchw(plan.tensor(y))


def check_op(got, ref, precision, tol=None, what=None):
    """The one-op bound of ``precision`` (OP_TOL), or ``tol`` in its place."""
    tol = OP_TOL[precision] if tol is None else tol
    if precision == "bf16":
        rel = ((got - ref).norm() / (ref.norm() + 1e-30)).item()
        assert rel <= tol, (what, rel)
    else:
        err = (got - ref).abs().max().item()
        scale = ref.abs().max().item() + 1e-30
        assert err <= tol * scale, (what, precision, err, scale, err / scale)


def match_rows(got, ref, tol=1e-3, box_tol=None):
    """got/ref: (K, C) detection rows of ONE image.  Rows are matched greedily on the bbox
    (first 4 columns) + score; returns (fraction of ref rows matched,
    fraction of elements within tol among matched rows)."""
    box_tol = tol if box_tol is None else box_tol
    used = np.zeros(len(got), bool)
    matched = 0; ok = 0; tot = 0
    for r in ref:
        d = np.abs(got[:, :5] - r[None, :5]).max(axis=1)
        d[used] = np.inf
        j = int(np.argmin(d))
        if d[j] <= box_tol:
            used[j] = True; matched += 1
            e = np.abs(got[j] - r) <= tol * np.maximum(1.0, np.abs(r))
            ok += int(e.sum()); tot += e.size
    return matched / max(1, len(ref)), (ok / tot if tot else 0.0)

"""CPU tests (-m "not gpu"): host-side logic, state_dict compatibility,
and the N>1 sharding/gather path on the gloo backend (world_size 2)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def test_product_path_refuses_cpu_tensors():
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    z = torch.zeros(1, 1, 8, 8)
    with pytest.raises(RuntimeError):
        multi_pose_decode(z, torch.zeros(1, 2, 8, 8), torch.zeros(1, 34, 8, 8), hm_hp=torch.zeros(1, 17, 8, 8))
    cfg = default_cfg("dla_34")
    with pytest.raises(RuntimeError):
        create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)(torch.zeros(1, 3, 64, 64))


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under centerpose_b200/ may reference it."""
    bad = []
    for dp, _, fns in os.walk(os.path.join(ROOT, "centerpose_b200")):
        for fn in fns:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, fn)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M) or "/root/reference" in txt:
                    bad.append(os.path.join(dp, fn))
    assert not bad, bad


def test_checkpoint_roundtrip_reference_format(tmp_path):
    """save_model / load_model keep the reference's file format (model.py:67-131), including the
    DataParallel 'module.' prefix and shape-mismatch tolerance."""
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model, load_model, save_model
    cfg = default_cfg("dla_34")
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
    p = str(tmp_path / "ck.pth")
    save_model(p, 7, m)
    ck = torch.load(p, weights_only=False)
    assert set(ck) == {"epoch", "state_dict"} and ck["epoch"] == 7
    assert "backbone_model.base.base_layer.0.weight" in ck["state_dict"]
    assert "head_model.hp_offset.2.bias" in ck["state_dict"]
    # DataParallel-style prefix + one mismatching tensor + one extra key
    sd = {"module." + k: v.clone() for k, v in ck["state_dict"].items()}
    sd["module.head_model.hm.2.weight"] = torch.zeros(3, 256, 1, 1)
    sd["module.extra.weight"] = torch.zeros(1)
    key = "module.backbone_model.base.level0.0.weight"
    sd[key] = torch.full_like(sd[key], 0.25)
    torch.save({"epoch": 3, "state_dict": sd}, p)
    m2 = load_model(create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg), p)
    assert float(m2.state_dict()["backbone_model.base.level0.0.weight"].mean()) == 0.25
    assert m2.state_dict()["head_model.hm.2.weight"].shape == (1, 256, 1, 1)


def test_post_process_matches_reference_golden():
    from centerpose_b200.image import multi_pose_post_process
    from oracle.post_process_ref import make_meta
    g = np.load(os.path.join(GOLD, "post_process.npz"))
    for case, ref in zip(g["cases"], g["out"]):
        meta = make_meta(int(case[0]), int(case[1]), float(case[2]), fix_res=bool(case[3]))
        out = multi_pose_post_process(g["dets"].copy(), [meta["c"]], [meta["s"]], meta["out_height"], meta["out_width"])
        out = np.array(out[0][1], dtype=np.float32).reshape(-1, 56)
        assert np.abs(out - ref).max() < 2e-3


def test_soft_nms_properties():
    from centerpose_b200.soft_nms import soft_nms_39
    rng = np.random.RandomState(0)
    n = 60
    xy = rng.uniform(0, 200, size=(n, 2)); wh = rng.uniform(20, 80, size=(n, 2))
    rows = np.zeros((n, 56), np.float32)
    rows[:, 0:2] = xy; rows[:, 2:4] = xy + wh; rows[:, 4] = rng.uniform(0.05, 1, size=n)
    rows[:, 5:] = rng.uniform(0, 1, size=(n, 51))
    before = rows.copy()
    keep = soft_nms_39(rows, Nt=0.5, method=2)
    assert 1 <= len(keep) <= n
    k = len(keep)
    assert rows[0, 4] == before[:, 4].max()                       # best row first, score untouched
    assert np.all(rows[:k, 4] >= 0.001)                           # survivors above threshold
    assert np.all(rows[:k, 4] <= before[:, 4].max() + 1e-6)
    assert np.array_equal(rows[:, 39:], before[:, 39:])           # kp-score columns never move (nms.pyx:214-217)
    iso = np.zeros((2, 56), np.float32); iso[0, :5] = [0, 0, 10, 10, 0.9]; iso[1, :5] = [100, 100, 110, 110, 0.8]
    soft_nms_39(iso, Nt=0.5, method=2)
    assert iso[0, 4] == np.float32(0.9) and iso[1, 4] == np.float32(0.8)   # disjoint boxes: no decay
    dup = np.zeros((2, 56), np.float32); dup[0, :5] = [0, 0, 10, 10, 0.9]; dup[1, :5] = [0, 0, 10, 10, 0.8]
    soft_nms_39(dup, Nt=0.5, method=2)
    assert abs(dup[1, 4] - 0.8 * np.exp(-1.0 / 0.5)) < 1e-6              # iou 1 -> exp(-1/sigma)


def test_cfg_defaults_and_yaml(tmp_path):
    from centerpose_b200.config import default_cfg, load_cfg
    cfg = default_cfg("dla_34")
    assert cfg.MODEL.HEAD_CONV == 256 and cfg["MODEL"]["INTERMEDIATE_CHANNEL"] == 64 and cfg.TEST.TOPK == 100
    y = tmp_path / "x.yaml"
    y.write_text("MODEL:\n  NAME: 'res_50'\n  HEAD_CONV: 64\nTEST:\n  TOPK: 50\n")
    c2 = load_cfg(str(y))
    assert c2.MODEL.NAME == "res_50" and c2.TEST.TOPK == 50 and c2.MODEL.DOWN_RATIO == 4


def test_plan_lowering_shapes():
    """The lowering walks the same graph as the reference: op census of DLA-34 (SURVEY Appendix A:
    45 base convs - 2 dead projects + 16 DCN offset convs + 12 head convs = 64 CONV + 1 STEM ...)."""
    from collections import Counter
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    cfg = default_cfg("dla_34")
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).set_precision("fp32")
    plan = m._plan(2, 128, 160, torch.device("cpu"))
    census = Counter(o.type for o in plan.ops)
    assert census == {1: 71 - 7, 2: 1, 3: 6, 4: 8, 5: 16}, census
    assert plan.out_shape == (32, 40)
    # the 16 DCN offset/mask convs are padded from 27 to 32 output channels (128-byte rows): count 27
    macs = sum(o.B * o.Ho * o.Wo * (27 if (o.flags & 4 and o.cout == 32) else o.cout) * o.kh * o.kw
               * sum(o.cin[j] for j in range(o.nsrc)) for o in plan.ops if o.type in (1, 2, 5)) / 2
    gmac_512 = macs / (128 * 160) * (512 * 512) / 1e9
    assert abs(gmac_512 - 40.17) < 0.1, gmac_512          # SURVEY: 40.24 incl. 0.067 dead project convs


def test_split_plane_helpers_and_packed_weight_scale():
    """Host side of the split-operand precisions (plan.py): hi = rn16(v), lo = rn16(v - hi) reproduces v to 2^-22 (fp16
    planes) / 2^-16 (bf16 planes); the fp16 weight pre-scale is an exact power of two that keeps the lo plane out of the
    subnormals; packed tensor-core weights keep hi + lo == w * scale; the accumulator compensation is linear in K."""
    import math
    from centerpose_b200.plan import PlanBuilder, pow2_scale, rz_compensation, split_planes
    g = torch.Generator().manual_seed(3)
    v = torch.randn(4096, generator=g) * torch.logspace(-2, 3, 4096)
    for dt, bits in ((torch.float16, 22), (torch.bfloat16, 16)):
        p = split_planes(v, dt)
        assert p.shape == (2, 4096) and p.dtype == dt
        rec = p[0].float() + p[1].float()
        assert ((rec - v).abs() <= v.abs() * 2.0 ** (-bits) * 1.01 + 1e-7).all()
        assert torch.equal(p[0], v.to(dt))
    sat = split_planes(torch.tensor([1e6, -1e6]), torch.float16)              # fp16 planes saturate instead of overflowing
    assert torch.isfinite(sat.float()).all() and sat[0].float().abs().max() == 65504.0
    for scale_in in (3e-4, 0.07, 1.0, 513.0):
        w = torch.randn(64, 32, 3, 3, generator=g) * scale_in
        s = pow2_scale(w)
        assert math.log2(s) == round(math.log2(s)) and 2.0 ** 12 <= float(w.abs().max()) * s < 2.0 ** 13
        lo = split_planes(w * s, torch.float16)[1].float()
        tiny = (lo != 0) & (lo.abs() < 2.0 ** -14)                                  # fp16 subnormal lo parts
        assert tiny.float().mean().item() < 1e-2                                   # only the weights that are themselves ~1e-4 of the largest
    assert pow2_scale(torch.zeros(3)) == 1.0
    assert rz_compensation("fp32", 576) == 1.0 and rz_compensation("bf16", 576) == 1.0
    c1, c2 = rz_compensation("fp16x2", 576) - 1.0, rz_compensation("fp16x2", 1152) - 1.0
    assert 0 < c1 < 1e-5 and abs(c2 - 2 * c1) < 1e-12
    pb = PlanBuilder(1, 32, 32, "fp16x2", torch.device("cpu"))
    w = torch.randn(48, 64, 3, 3, generator=g) * 0.05
    packed, sc = pb._pack_conv_tc(w, 64)                                            # [plane][tap][slab][Co_pad][bk]
    assert sc == pow2_scale(w) and pb._acc_scale(576, sc) == rz_compensation("fp16x2", 576) / sc
    rec = (packed[0].float() + packed[1].float())[:, 0, :48, :]                     # [tap][Co][Ci]
    ref = (w * sc).permute(2, 3, 0, 1).reshape(9, 48, 64)
    assert (rec - ref).abs().max().item() <= ref.abs().max().item() * 2.0 ** -21


def test_stride2_stem_space_to_depth_lowering_is_the_same_convolution():
    """Split precisions lower a k x k / stride-2 stem to CPB200_OP_S2D + a stride-1 conv over 16 channels (plan.py::stem).
    The lowering is pure index arithmetic: replay it with torch on the CPU — space-to-depth of the image, the repacked weights
    the builder emitted — and compare with the strided convolution it replaces (msra_resnet.py:116-117, pose_higher_hrnet.py:283)."""
    import torch.nn.functional as F
    from centerpose_b200.plan import OP_S2D, PlanBuilder
    g = torch.Generator().manual_seed(5)
    for k, co, H, W in ((7, 64, 20, 28), (3, 64, 16, 24), (3, 16, 12, 20)):
        x = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64)
        w = torch.randn(co, 3, k, k, generator=g, dtype=torch.float64)
        b = torch.randn(co, generator=g, dtype=torch.float64)
        pb = PlanBuilder(2, H, W, "fp16x2", torch.device("cpu"))
        y = pb.stem(pb.input(3), w.float(), b.float(), k, 2, k // 2, relu=False)
        assert [o.type for o in pb.ops] == [OP_S2D, 1]
        conv = pb.ops[1]
        k2 = (k + 1) // 2 + 1
        assert conv.k == (k2, k2) and conv.stride == 1 and conv.pad == (k2 // 2, k2 // 2) and (y.C, y.H, y.W) == (co, H // 2, W // 2)
        # z[b, (py*2+px)*3 + c, h, w] = x[b, c, 2h+py, 2w+px], channels 12..15 zero (include/centerpose_b200.h, CPB200_OP_S2D)
        z = torch.zeros(2, 16, H // 2, W // 2, dtype=torch.float64)
        for py in range(2):
            for px in range(2):
                z[:, (py * 2 + px) * 3:(py * 2 + px) * 3 + 3] = x[:, :, py::2, px::2]
        got = F.conv2d(z, conv.w_raw.double(), b, stride=1, padding=k2 // 2)
        ref = F.conv2d(x, w.float().double(), b, stride=2, padding=k // 2)
        assert got.shape == ref.shape and (got - ref).abs().max().item() < 1e-9, (k, (got - ref).abs().max().item())
    # odd sizes keep the strided stem op
    pb = PlanBuilder(2, 21, 28, "fp16x2", torch.device("cpu"))
    pb.stem(pb.input(3), torch.randn(64, 3, 7, 7), torch.zeros(64), 7, 2, 3)
    assert pb.ops[0].type == 2


_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from centerpose_b200.sharding import shard_range, gather_detections
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
B = 10
lo, hi = shard_range(B, rank, 2)
assert (lo, hi) == ((0, 5) if rank == 0 else (5, 10))
full = torch.arange(B * 3 * 4, dtype=torch.float32).view(B, 3, 4)
out = gather_detections(full[lo:hi].clone(), group=None)
assert torch.equal(out, full), out
# ragged split
lo, hi = shard_range(7, rank, 2)
out = gather_detections(full[:7][lo:hi].clone(), group=None, total=7)
assert torch.equal(out, full[:7])
dist.destroy_process_group()
print("ok", rank)
'''


def test_sharding_world_size_2_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    port = str(29500 + (os.getpid() % 2000))
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=180)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_soft_nms_matches_compiled_reference_golden():
    """``soft_nms_39`` port vs golden vectors produced by the reference's own Cython module compiled in the build
    container (oracle/build_ref.py, lib/external/nms.pyx:172-275): identical keep counts and row movements; scores
    within 1 float ulp (2e-7) — the reference built with Cython 3 evaluates its ``+ 1`` / ``1 - ov`` terms in double
    (int literals become ``1.0``), the port keeps C ``float`` like the original Cython 0.29 build."""
    from centerpose_b200.soft_nms import soft_nms_39
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "soft_nms.npz"))
    for boxes, out, keep, prm in zip(g["boxes"], g["out"], g["keep"], g["params"]):
        N, method, Nt, thr = int(prm[0]), int(prm[1]), float(prm[2]), float(prm[3])
        rows = boxes[:N].copy()
        k = soft_nms_39(rows, sigma=0.5, Nt=Nt, threshold=thr, method=method)
        assert len(k) == int(keep)
        assert np.abs(rows - out[:N]).max() <= 2e-7


def test_convert_eval_format_matches_reference_statement():
    """coco_format.convert_eval_format vs a literal restatement of lib/datasets/coco_hp.py:56-83 (the reference method
    lives on a dataset class that needs pycocotools + annotation files)."""
    from centerpose_b200.coco_format import convert_eval_format

    def ref(all_bboxes):                                   # coco_hp.py:56-83, verbatim semantics
        to_float = lambda x: float("{:.2f}".format(x))
        detections = []
        for image_id in all_bboxes:
            for dets in all_bboxes[image_id][1]:
                bbox = dets[:4]
                bbox[2] -= bbox[0]; bbox[3] -= bbox[1]
                score = dets[4]
                prob = np.array(np.array(dets[39:56]) > 0.1).astype(np.int32).reshape(17, 1)
                kps = np.array(dets[5:39], dtype=np.float32).reshape(-1, 2)
                pred = list(map(to_float, np.concatenate([kps, prob], axis=1).reshape(51).tolist()))
                detections.append({"image_id": int(image_id), "category_id": 1, "bbox": list(map(to_float, bbox)),
                                   "score": float("{:.2f}".format(score)), "keypoints": pred})
        return detections

    rng = np.random.RandomState(4)
    res = {}
    for img in (17, 42):
        rows = rng.uniform(0, 640, size=(5, 56)); rows[:, 2:4] += rows[:, 0:2]; rows[:, 4] = rng.uniform(0, 1, 5)
        rows[:, 39:] = rng.uniform(0, 0.3, size=(5, 17))
        res[img] = {1: rows.astype(np.float32).tolist()}
    import copy
    assert convert_eval_format(copy.deepcopy(res)) == ref(copy.deepcopy(res))

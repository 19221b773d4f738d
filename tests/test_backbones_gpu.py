"""Every network-level GPU check of the seven backbones (DLA-34, ResNet-50, HRNet-W32, MobileNetV3, HarDNet,
MobileNetV2, GhostNet), as tables: each row is one (backbone, input, precision) combination and its bound.  The weights
are the conditioned seed-317 ones (oracle/init_recipe.py); the goldens are the unmodified reference's own fp32 outputs
on the same weights and images (oracle/make_golden.py).

Tolerances (floating point; this docstring is the one statement of the network bounds):
  head maps vs golden (MAPS), max|err| / max|ref| and relative L2, maps subsampled by the golden's stride:
    fp32, fp16x2 : 5e-4 and 2e-4 on all 16 goldens (the conditioned-init network amplifies perturbations x1.7; the
                   reference's own fp32 CPU result is 2e-6 from a float64 evaluation; fp16x2 measures ~5e-6)
    bf16x2       : 2e-3 and 5e-4 on the DLA-34 / ResNet-50 / HRNet / MobileNetV3 goldens; 5e-3 and 2e-3 on MobileNetV2
                   and GhostNet (16 significand bits per plane)
    bf16         : relative L2 only, 4e-2 (GhostNet: 1.1e-2 measured); MobileNetV2 1.5e-1 (7.6e-2 at 96x160, 1.0e-1 at
                   512x512 measured on an H100: plain bf16 activations through 52 narrow layers).  bf16 is the fast mode,
                   with no parity claim
  against the oracle's forward (ORACLE): DLA-34 fp32 5e-4 and 2e-4; bf16 on the CUDA-core and the wgmma kernels
                   relative L2 3e-2 (MobileNetV3 4e-2)
  decoded rows at 512x512 (ROWS): rows matched greedily on bbox + score within box_tol (top-K is discontinuous: two
                   peaks closer than the logit error swap rows), then each value within 1e-3 * max(1, |ref|) on the
                   matched rows (tests/util.py::match_rows).  fp32 (CUDA-core summation order) >= 90 % of the rows and
                   >= 97 % of the values; fp16x2 >= 99 % / 99 %, all rows and all values for MobileNetV2 and GhostNet,
                   all rows and >= 99.9 % of the values for HarDNet (a near-tie, see ROWS); bf16x2 >= 90 % / 95 %;
                   bf16 DLA-34 >= 20 % of the rows within half an output pixel, the other bf16 statistics reported
  batch consistency (BATCH): bit for bit
"""
import os

import numpy as np
import pytest
import torch

from tests.util import DEV, GOLD, golden_check, golden_input, match_rows, model

pytestmark = pytest.mark.gpu

ARCH = {"dla34": "dla_34", "res50": "res_50", "hrnet32": "hrnet", "mbv3": "mobilenetv3", "hardnet": "hardnet",
        "mbv2": "mobilenetv2", "ghostnet": "ghostnet"}
GOLDENS = ["dla34_128", "dla34_96x160", "dla34_512", "res50_128", "res50_512", "hrnet32_128", "hrnet32_256x320",
           "hrnet32_512", "mbv3_128x160", "mbv3_512", "hardnet_128", "hardnet_96x160", "hardnet_512", "mbv2_512",
           "mbv2_96x160", "ghostnet_512"]
SPLIT4 = ["dla34_128", "dla34_96x160", "dla34_512", "res50_128", "res50_512", "hrnet32_128", "hrnet32_256x320",
          "hrnet32_512", "mbv3_128x160", "mbv3_512"]

# (golden, precision, max|err| / max|ref|, relative L2); None: not bounded
MAPS = ([(t, "fp32", 5e-4, 2e-4) for t in GOLDENS]
        + [(t, "fp16x2", 5e-4, 2e-4) for t in GOLDENS]
        + [(t, "bf16x2", 2e-3, 5e-4) for t in SPLIT4]
        + [(t, "bf16x2", 5e-3, 2e-3) for t in ("mbv2_512", "mbv2_96x160", "ghostnet_512")]
        + [(t, "bf16", None, 4e-2) for t in ("res50_512", "hrnet32_512", "mbv3_512", "hardnet_512", "ghostnet_512")]
        + [(t, "bf16", None, 1.5e-1) for t in ("mbv2_512", "mbv2_96x160")]
        + [("dla34_512", "bf16", None, None)])          # its decoded rows are bounded (ROWS)

# (golden, precision) -> (fraction of rows matched, fraction of values within 1e-3 on them, box_tol); None: reported
ROWS = {**{(t, "fp32"): (0.9, 0.97, 2e-2) for t in ("dla34_512", "res50_512", "hrnet32_512", "mbv3_512", "hardnet_512",
                                                    "mbv2_512", "ghostnet_512")},
        **{(t, "fp16x2"): (0.99, 0.99, 2e-2) for t in ("dla34_512", "res50_512", "hrnet32_512", "mbv3_512")},
        # All 100 rows match.  Values: >= 99.9 %, not 100 %.  Keypoint 1 of reference row 98 sits on a near-tie of the
        # decode's keypoint-heat-map snapping.  Perturbing the reference's exact head maps by 2e-6 relative noise moves
        # that keypoint to the other candidate in 3 of 5 seeds.  The fp32 CUDA-core path (maps 3e-7 from the reference)
        # and fp16x2 (1.5e-6) both land on the other candidate: 2 of 5 600 values.
        ("hardnet_512", "fp16x2"): (1.0, 0.999, 2e-2),
        ("mbv2_512", "fp16x2"): (1.0, 1.0, 2e-2),
        ("ghostnet_512", "fp16x2"): (1.0, 1.0, 2e-2),
        **{(t, "bf16x2"): (0.9, 0.95, 2e-2) for t in ("dla34_512", "res50_512", "hrnet32_512", "mbv3_512")},
        # measured: 37 % of the reference rows have a counterpart within half a pixel, 12 % of their values are within
        # 1e-3 — plain bf16 is a fast mode, NOT the parity-qualified one (that is 'fp16x2')
        ("dla34_512", "bf16"): (0.2, None, 0.5),
        **{(t, "bf16"): (None, None, 0.5) for t in ("res50_512", "hrnet32_512", "mbv3_512")}}

# (golden, precision) whose program must hold no CONVERT op (no fp32 island)
NO_CONVERT = {("hardnet_512", "fp16x2")}


@pytest.mark.parametrize("tag,precision,max_tol,rel_tol", MAPS, ids=[f"{t}-{p}" for t, p, _, _ in MAPS])
def test_head_maps_match_golden(tag, precision, max_tol, rel_tol):
    """Whole network against the unmodified reference's head maps; at 512x512 the decoded rows too.  Small inputs also
    exercise the fp32 islands of the split precisions (maps < 8 pixels wide, HRNet's upsample-add, MobileNetV3's
    depthwise / SE ops, HarDNet's 2x2 deepest map and odd pools, the stride-2 stem)."""
    m, _ = model(ARCH[tag.rsplit("_", 1)[0]], precision)
    _, mx, rel, rows = golden_check(m, tag)
    print(f"{tag} {precision}: max/max {mx:.3e} relL2 {rel:.3e}")
    assert max_tol is None or mx <= max_tol, (mx, rel)
    assert rel_tol is None or rel <= rel_tol, (mx, rel)
    if (tag, precision) in ROWS:
        min_rows, min_elems, box_tol = ROWS[(tag, precision)]
        r, e = match_rows(*rows, tol=1e-3, box_tol=box_tol)
        print(f"{tag} {precision}: rows matched within {box_tol} {r:.3f}, elements within 1e-3 {e:.4f}")
        assert min_rows is None or r >= min_rows, (r, e)
        assert min_elems is None or e >= min_elems, (r, e)
    if (tag, precision) in NO_CONVERT:
        from centerpose_b200.plan import OP_CONVERT
        plan = next(iter(m._plans.values()))
        assert sum(o.type == OP_CONVERT for o in plan.ops) == 0


# (arch, golden whose input is used, fp32 bound (max|err| / max|ref|, relative L2), bf16 relative L2); golden None:
# synth_images(2, 128, 160, seed=5)
ORACLE = [("dla_34", None, (5e-4, 2e-4), 3e-2), ("res_50", "res50_128", None, 3e-2), ("hrnet", "hrnet32_128", None, 3e-2),
          ("hrnet", "hrnet32_256x320", None, 3e-2), ("mobilenetv3", "mbv3_128x160", None, 4e-2)]


@pytest.mark.parametrize("arch,tag,fp32_tol,bf16_tol", ORACLE, ids=[f"{a}-{t or 'seed5'}" for a, t, _, _ in ORACLE])
def test_forward_matches_oracle(arch, tag, fp32_tol, bf16_tol):
    """The forward against the oracle's (oracle/dla_ref.py) on the same weights: bf16 activations on the CUDA-core
    kernels, then on the wgmma kernels.  HRNet at 128x128 drives the lowest-resolution branches (4x4, 8x8) through the
    CUDA-core fallbacks; 256x320 keeps every conv on the wgmma kernels."""
    from oracle import dla_ref
    from oracle.init_recipe import synth_images
    x = synth_images(2, 128, 160, seed=5) if tag is None else golden_input(tag)
    m, sd = model(arch, "fp32")
    ref = torch.cat(dla_ref.forward(sd, x, arch=arch), dim=1)
    if fp32_tol is not None:
        got = torch.cat(m(x.to(DEV)), dim=1).cpu().double(); r = ref.double()
        mx = ((got - r).abs().max() / r.abs().max()).item(); rel = ((got - r).norm() / r.norm()).item()
        assert mx <= fp32_tol[0] and rel <= fp32_tol[1], (mx, rel)
    for tc in (False, True):
        m.set_precision("bf16", tc=tc)
        got16 = torch.cat(m(x.to(DEV)), dim=1).cpu()
        rel = ((got16 - ref).norm() / ref.norm()).item()
        assert rel <= bf16_tol, (tc, rel)


# (arch, precision, batch): the bf16 batches are the benchmark's per-backbone sizes
BATCH = [("dla_34", "bf16", 32), ("res_50", "bf16", 16), ("hrnet", "bf16", 16), ("mobilenetv3", "bf16", 64),
         ("hardnet", "bf16", 64), ("dla_34", "fp16x2", 3)]


@pytest.mark.parametrize("arch,precision,B", BATCH, ids=[f"{a}-{p}-{b}" for a, p, b in BATCH])
def test_batch_consistency_and_output_rebinding(arch, precision, B):
    """(1) Image i of a batch equals the same image run alone, bit for bit (tiles never mix images).  (2) The
    tensor-core ops read dst / res / bias from the live op at every launch: a second forward on the SAME plan while the
    first call's outputs are still held must return independent, correct tensors (an earlier bug: `Plan.bind`
    re-pointed ops[i].dst after the one-time prepare had cached it)."""
    from oracle.init_recipe import synth_images
    m, _ = model(arch, precision)
    x1 = synth_images(B, 128, 160, seed=21).to(DEV)
    x2 = synth_images(B, 128, 160, seed=22).to(DEV)
    ref1 = [t.clone() for t in m(x1)]
    m.invalidate()
    ref2 = [t.clone() for t in m(x2)]
    m.invalidate()
    o1 = m(x1)
    o2 = m(x2)                       # same plan, o1 still alive
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
            assert torch.equal(a[i:i + 1], b), (arch, i)


def test_forward_rejects_cpu_and_training():
    m, _ = model("dla_34", "bf16")
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 64, 64))
    m.train()
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 64, 64, device=DEV))


def _detector(arch):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg(arch)
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    return det


def test_hardnet_detector_run_batch_fused():
    from oracle import post_process_ref
    det = _detector("hardnet")
    x = torch.randn(2, 3, 512, 512, generator=torch.Generator().manual_seed(1))
    out = det.run_batch_fused(x, [post_process_ref.make_meta(480, 640), post_process_ref.make_meta(512, 512)])
    assert out.shape == (2, 100, 56) and np.isfinite(out).all()
    assert (out[:, :, 4] > 0).all()


@pytest.mark.parametrize("arch,tag", [("mobilenetv2", "mbv2_512"), ("ghostnet", "ghostnet_512")])
def test_detector_run_batch_fused_matches_reference_rows(arch, tag):
    """run_batch_fused (fp16x2 forward + decode + back-projection on the device) against the reference's decoded rows
    of its own maps, back-projected by the oracle's post-process, for a 512x512 image."""
    from oracle import post_process_ref
    from oracle.init_recipe import synth_images
    g = np.load(os.path.join(GOLD, f"{tag}.npz"))
    det = _detector(arch)
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
    det = _detector(arch)
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, (480, 640, 3), dtype=np.uint8), rng.integers(0, 256, (512, 512, 3), dtype=np.uint8)]
    res = det.run_images(imgs)
    assert len(res) == 2
    for r in res:
        r = np.asarray(r)
        assert r.ndim == 2 and r.shape[1] == 56 and len(r) > 0 and np.isfinite(r).all()

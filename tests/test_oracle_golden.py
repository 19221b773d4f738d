"""CPU tests: the oracle restatements replay the golden vectors that
``oracle/make_golden.py`` produced by running the unmodified reference (pinning)."""
import glob
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import dcn_ref, decode_ref, dla_ref, post_process_ref
from oracle.init_recipe import conditioned_state_dict, synth_images

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


DECODE_FILES = sorted(glob.glob(os.path.join(GOLD, "decode_*.npz")))


@pytest.mark.parametrize("path", DECODE_FILES, ids=[os.path.basename(p)[7:-4] for p in DECODE_FILES])
def test_decode_oracle_matches_reference_golden(path):
    g = np.load(path)
    B, H, W, K, seed, use_reg, use_off = [int(v) for v in g["meta"]]
    inp = decode_ref.synth_decode_inputs(B, H, W, seed=seed, kind=str(g["kind"]))
    assert _sha(*[inp[k] for k in sorted(inp)]) == str(g["input_sha"]), "synthetic input drifted"
    det = decode_ref.multi_pose_decode(inp["heat"], inp["wh"], inp["kps"],
                                       inp["reg"] if use_reg else None, inp["hm_hp"],
                                       inp["hp_offset"] if use_off else None, K=K)
    ref = g["det"]
    assert det.shape == ref.shape == (B, K, 56)
    pos = ref[:, :, 4] > 0          # rows with score 0 are arbitrary zero-cells in the reference
    assert np.array_equal(det[pos], ref[pos])     # bit-exact (fp32, same operation order)


def test_decode_requires_hm_hp_like_reference():
    inp = decode_ref.synth_decode_inputs(1, 16, 16, seed=1)
    with pytest.raises(NameError):
        decode_ref.multi_pose_decode(inp["heat"], inp["wh"], inp["kps"], inp["reg"], None, None, K=10)


def test_decode_k_larger_than_map_raises():
    inp = decode_ref.synth_decode_inputs(1, 4, 4, seed=1)
    with pytest.raises(RuntimeError):
        decode_ref.multi_pose_decode(**inp, K=100)


def test_dcn_restatements_match_golden():
    g = np.load(os.path.join(GOLD, "dcn_small.npz"))
    lit = dcn_ref.dcn_v2_forward_loops(g["x"], g["w"], g["b"], g["off"], g["msk"])
    vec = dcn_ref.dcn_v2_forward(*[torch.from_numpy(g[k]) for k in ("x", "w", "b", "off", "msk")]).numpy()
    assert np.abs(lit - g["out"]).max() < 1e-5
    assert np.abs(vec - g["out"]).max() < 1e-5


def test_dcn_zero_offset_known_answer():
    """DCNv2/test.py:31-66 check_zero_offset: identity 3x3 weights, zero offsets,
    mask = sigmoid(0) = 0.5  =>  2 * DCNv2(x) == x."""
    C = 4
    x = torch.randn(2, C, 9, 11, generator=torch.Generator().manual_seed(0))
    w = torch.zeros(C, C, 3, 3)
    for c in range(C):
        w[c, c, 1, 1] = 1.0
    off = torch.zeros(2, 18, 9, 11); msk = torch.full((2, 9, 9, 11), 0.5)
    out = dcn_ref.dcn_v2_forward(x, w, torch.zeros(C), off, msk)
    assert (2 * out - x).abs().max().item() < 1e-10
    out_l = dcn_ref.dcn_v2_forward_loops(x.numpy(), w.numpy(), np.zeros(C), off.numpy(), msk.numpy())
    assert np.abs(2 * out_l - x.numpy()).max() < 1e-10


def test_dcn_module_matches_torchvision():
    tv = pytest.importorskip("torchvision.ops")
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 8, 10, 12, generator=g)
    w = torch.randn(6, 8, 3, 3, generator=g) * 0.2; b = torch.randn(6, generator=g)
    ow = torch.randn(27, 8, 3, 3, generator=g) * 0.2; ob = torch.randn(27, generator=g)
    mine = dcn_ref.dcn_module_forward(x, w, b, ow, ob)
    om = torch.nn.functional.conv2d(x, ow, ob, padding=1)
    o1, o2, m = torch.chunk(om, 3, dim=1)
    ref = tv.deform_conv2d(x, torch.cat((o1, o2), 1), w, b, padding=1, mask=torch.sigmoid(m))
    assert (mine - ref).abs().max().item() < 1e-4


def test_post_process_matches_golden():
    g = np.load(os.path.join(GOLD, "post_process.npz"))
    for case, ref in zip(g["cases"], g["out"]):
        h, w, scale, fix = int(case[0]), int(case[1]), float(case[2]), bool(case[3])
        meta = post_process_ref.make_meta(h, w, scale, fix_res=fix)
        out = post_process_ref.multi_pose_post_process(g["dets"].copy(), [meta["c"]], [meta["s"]],
                                                       meta["out_height"], meta["out_width"])[0][1]
        assert np.abs(out - ref).max() < 2e-3      # image pixels, values up to ~2000


@pytest.mark.parametrize("tag", ["128", "96x160"])
def test_dla34_oracle_matches_golden(tag):
    g = np.load(os.path.join(GOLD, f"dla34_{tag}.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    from centerpose_b200.model import create_model
    from centerpose_b200.config import default_cfg
    cfg = default_cfg("dla_34")
    tmpl = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).state_dict()
    sd = conditioned_state_dict(tmpl, 317)
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(g["sd_sha"])
    x = synth_images(B, H, W, seed=317)
    assert _sha(x.numpy()) == str(g["x_sha"])
    maps = torch.cat(dla_ref.forward(sd, x), dim=1).numpy()
    ref = g["maps"]
    assert maps.shape == ref.shape
    assert np.abs(maps - ref).max() <= 1e-4 * np.abs(ref).max()


def test_res50_oracle_matches_golden():
    g = np.load(os.path.join(GOLD, "res50_128.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    from centerpose_b200.model import create_model
    from centerpose_b200.config import default_cfg
    cfg = default_cfg("res_50")
    sd = conditioned_state_dict(create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).state_dict(), 317)
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(g["sd_sha"])
    x = synth_images(B, H, W, seed=317)
    maps = torch.cat(dla_ref.forward(sd, x, arch="res_50"), dim=1).numpy()
    assert np.abs(maps - g["maps"]).max() <= 1e-4 * np.abs(g["maps"]).max()


def test_hrnet_oracle_matches_golden():
    """HRNet-W32 (BASELINE config 4): oracle restatement vs the reference module's golden maps; also pins that the
    product's parameter tree has exactly the reference's key names (the recipe draws in sorted-key order)."""
    g = np.load(os.path.join(GOLD, "hrnet32_128.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    from centerpose_b200.model import create_model
    from centerpose_b200.config import default_cfg
    cfg = default_cfg("hrnet")
    sd = conditioned_state_dict(create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).state_dict(), 317)
    assert len(sd) == 1776
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(g["sd_sha"])
    x = synth_images(B, H, W, seed=317)
    maps = torch.cat(dla_ref.forward(sd, x, arch="hrnet"), dim=1).numpy()
    assert np.abs(maps - g["maps"]).max() <= 1e-4 * np.abs(g["maps"]).max()


def test_mobilenetv3_oracle_matches_golden():
    """MobileNetV3 + DCN IDAUp (BASELINE config 5): oracle restatement vs the reference module's golden maps."""
    g = np.load(os.path.join(GOLD, "mbv3_128x160.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    from centerpose_b200.model import create_model
    from centerpose_b200.config import default_cfg
    cfg = default_cfg("mobilenetv3")
    sd = conditioned_state_dict(create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).state_dict(), 317)
    assert len(sd) == 471
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(g["sd_sha"])
    x = synth_images(B, H, W, seed=317)
    maps = torch.cat(dla_ref.forward(sd, x, arch="mobilenetv3"), dim=1).numpy()
    assert np.abs(maps - g["maps"]).max() <= 1e-4 * np.abs(g["maps"]).max()


AR_TAGS = {"dla34": ("dla_34", "dla_34"), "res50": ("res_50", "res_50"), "hrnet32": ("hrnet", "hrnet"),
           "hrnet48": ("hrnet_w48", "hrnet"), "mbv3": ("mobilenetv3", "mobilenetv3"), "hardnet": ("hardnet", None),
           "mbv2": ("mobilenetv2", None), "ghostnet": ("ghostnet", None)}


@pytest.mark.parametrize("name", sorted(AR_TAGS))
def test_oracle_matches_extreme_aspect_golden(name):
    """Every configuration at the 96x640 input of tests/golden/<name>_96x640.npz (oracle/make_golden.py: gen_aspect):
    deep maps 3x20 and 1x10.  Also pins that the product's parameter tree of each configuration (HRNet-W48 included)
    draws the reference's weights."""
    from centerpose_b200.model import create_model
    from oracle import ghostnet_ref, hardnet_ref, mobilenetv2_ref
    from tests.util import config
    arch, oracle_arch = AR_TAGS[name]
    g = np.load(os.path.join(GOLD, f"{name}_96x640.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    st = int(g["stride"])
    cfg = config(arch)
    sd = conditioned_state_dict(create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).state_dict(), 317)
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(g["sd_sha"])
    x = synth_images(B, H, W, seed=317)
    assert _sha(x.numpy()) == str(g["x_sha"])
    if oracle_arch is not None:
        out = dla_ref.forward(sd, x, arch=oracle_arch)
    else:
        out = {"hardnet": hardnet_ref, "mobilenetv2": mobilenetv2_ref, "ghostnet": ghostnet_ref}[arch].forward(sd, x)
    maps = torch.cat(out, dim=1).numpy()[:, :, ::st, ::st]
    assert maps.shape == g["maps"].shape
    assert np.abs(maps - g["maps"]).max() <= 1e-4 * np.abs(g["maps"]).max()

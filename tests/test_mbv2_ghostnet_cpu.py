"""CPU tests (-m "not gpu") of the MobileNetV2 and GhostNet backbones (centerpose_b200/archs/mobilenetv2.py,
centerpose_b200/archs/ghostnet.py): the oracles against the reference-generated goldens, the parameter trees' key
names / shapes / order, the lowerings' op census and flags, and the reference checkpoint format."""
import os
from collections import Counter

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ARCHS = {"mobilenetv2": ("mobilenetv2_512x512", 354), "ghostnet": ("ghost_net", 502)}
GOLDENS = [("mobilenetv2", "mbv2_512"), ("mobilenetv2", "mbv2_96x160"), ("ghostnet", "ghostnet_512")]


def _sha(*arrays):
    import hashlib
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _model(arch, name=None):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    cfg = default_cfg(arch)
    return create_model(name or cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg), cfg


def _oracle(arch):
    from oracle import ghostnet_ref, mobilenetv2_ref
    return mobilenetv2_ref if arch == "mobilenetv2" else ghostnet_ref


@pytest.mark.parametrize("arch,tag", GOLDENS)
def test_oracle_matches_reference_golden(arch, tag):
    """oracle/{mobilenetv2,ghostnet}_ref.py restate the reference's forward; the goldens are the unmodified reference's
    own backbone features and head maps (the generator pins the oracles to 0 difference)."""
    from oracle.init_recipe import conditioned_state_dict, synth_images
    g = np.load(os.path.join(GOLD, f"{tag}.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    st, fst = int(g["stride"]), int(g["feat_stride"])
    m, _ = _model(arch)
    sd = conditioned_state_dict(m.state_dict(), 317)
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(g["sd_sha"])
    x = synth_images(B, H, W, 317)
    assert _sha(x.numpy()) == str(g["x_sha"])
    ora = _oracle(arch)
    sdf = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    backbone = ora.mobilenetv2_backbone if arch == "mobilenetv2" else ora.ghostnet_backbone
    with torch.no_grad():
        feat = backbone(sdf, x).numpy()[:, :, ::fst, ::fst]
    maps = torch.cat(ora.forward(sd, x), dim=1).numpy()[:, :, ::st, ::st]
    assert feat.shape == g["feat"].shape and maps.shape == g["maps"].shape
    assert np.abs(feat - g["feat"]).max() <= 1e-4 * np.abs(g["feat"]).max()
    assert np.abs(maps - g["maps"]).max() <= 1e-4 * np.abs(g["maps"]).max()


@pytest.mark.parametrize("arch", sorted(ARCHS))
def test_state_dict_matches_reference(arch):
    """354 (MobileNetV2) / 502 (GhostNet) backbone entries + 24 head tensors, in the reference module's order with its
    shapes.  Without the reference the golden's weight sha still pins every key name and shape (the recipe draws in
    sorted-key order)."""
    from oracle.init_recipe import conditioned_state_dict
    from oracle.ref_harness import reference_available
    yaml, n_backbone = ARCHS[arch]
    m, _ = _model(arch)
    own = m.state_dict()
    assert sum(k.startswith("backbone_model.") for k in own) == n_backbone and len(own) == n_backbone + 24
    tag = "mbv2_512" if arch == "mobilenetv2" else "ghostnet_512"
    sd = conditioned_state_dict(own, 317)
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == \
        str(np.load(os.path.join(GOLD, f"{tag}.npz"))["sd_sha"])
    if not reference_available():
        pytest.skip("the reference is not mounted: key order and shapes checked through the golden's sha only")
    from oracle.ref_harness import ref_create_model
    ref, _ = ref_create_model(yaml)
    rsd = ref.state_dict()
    assert list(rsd) == list(own)
    assert all(tuple(rsd[k].shape) == tuple(own[k].shape) for k in rsd)


def test_channel_tables():
    from centerpose_b200.archs import ghostnet as gh
    from centerpose_b200.archs import mobilenetv2 as mb2
    feats, chans = mb2.layout()
    assert chans == [16, 16, 48, 160] and [len(b) for _, _, b in feats] == [3, 3, 7, 4]
    assert feats[0][2][0] == (16, 16, 8, 1, 1)                     # the t = 1 block: 16 -> 8 channels
    blocks = gh.blocks()
    assert len(blocks) == 16 and gh.FEAT_C == 160
    # ghost-module halves are multiples of 4, mostly not of 16
    assert sorted({h // 2 for _, _, _, h, _, _, _ in blocks}) == [8, 24, 36, 60, 92, 100, 120, 240, 336, 480]


@pytest.mark.parametrize("name", ["mobilenetv2", "mobilenetv2_10", "mobilenetv2_5", "ghostnet", "ghostnet_1"])
def test_create_model_accepts_any_suffix(name):
    """create_model no longer raises KeyError; like the reference, the _N suffix does not change the network
    (MobileNetV2 is always width 0.5)."""
    arch = name.split("_")[0]
    m, cfg = _model(arch, name)
    ref, _ = _model(arch)
    assert [(k, v.shape) for k, v in m.state_dict().items()] == [(k, v.shape) for k, v in ref.state_dict().items()]
    assert cfg.MODEL.HEAD_CONV == 256
    assert cfg.MODEL.INTERMEDIATE_CHANNEL == (24 if arch == "mobilenetv2" else 160)


def test_unknown_backbone_message_lists_the_new_ones():
    with pytest.raises(KeyError, match="mobilenetv2, ghostnet"):
        _model("dla_34", "efficientdet")


def test_fold_bn_eps():
    """MobileNetUp's BatchNorms use eps 1e-3; fold_bn takes it as an argument (default 1e-5)."""
    from centerpose_b200.plan import fold_bn
    w = torch.randn(4, 3, 1, 1)
    bnd = {"weight": torch.rand(4) + 0.5, "bias": torch.randn(4), "running_mean": torch.randn(4),
           "running_var": torch.rand(4) * 1e-3}
    x = torch.randn(2, 3, 5, 5)
    for eps in (1e-5, 1e-3):
        wf, bf = fold_bn(w, None, bnd, eps=eps)
        ref = torch.nn.functional.batch_norm(torch.nn.functional.conv2d(x, w), bnd["running_mean"], bnd["running_var"],
                                             bnd["weight"], bnd["bias"], False, 0.0, eps)
        assert torch.allclose(torch.nn.functional.conv2d(x, wf, bf), ref, rtol=1e-5, atol=1e-5)


def _plan(arch, precision, B, H, W):
    m, _ = _model(arch)
    m.set_precision(precision)
    return m._plan(B, H, W, torch.device("cpu"))


def test_mobilenetv2_plan_census():
    """fp32 lowering on the CPU: ReLU6 on the stem, the 16 expand convs and the 17 depthwise convs; the three IDAUp
    steps are DWDECONV_ADD ops in the bias form (k 2, stride 2, pad 0, ReLU, a skip); every activation is a multiple
    of 16 channels; the heads run at stride 4."""
    from centerpose_b200.plan import (FLAG_RELU, FLAG_RELU6, OP_CONV, OP_DWCONV, OP_DWDECONV_ADD, OP_STEM)
    plan = _plan("mobilenetv2", "fp32", 2, 96, 160)
    ops = plan.pb.ops
    census = Counter(o.type for o in ops)
    assert plan.out_shape == (24, 40)
    assert census == {OP_STEM: 1, OP_DWCONV: 17, OP_DWDECONV_ADD: 3, OP_CONV: 16 + 17 + 1 + 3 + 1 + 12}, census
    assert sum(bool(o.flags & FLAG_RELU6) for o in ops) == 1 + 16 + 17
    assert all(o.flags & FLAG_RELU6 for o in ops if o.type in (OP_STEM, OP_DWCONV))
    ups = [o for o in ops if o.type == OP_DWDECONV_ADD]
    assert all(o.k == (2, 2) and o.stride == 2 and o.pad == (0, 0) and o.flags == FLAG_RELU and o.bias is not None
               and o.extra[0] is not None and o.srcs[0].C == 32 for o in ups)
    assert [(o.dst.H, o.dst.W) for o in ups] == [(6, 10), (12, 20), (24, 40)]
    assert all(s.C % 16 == 0 for o in ops if o.type != OP_STEM for s in o.srcs)


def test_ghostnet_plan_census():
    """fp32 lowering on the CPU: 32 ghost modules (a 1x1 conv + a depthwise op each), the SE gates' second FC with the
    clip01 epilogue (one per slab: 7 SE layers x 2), ten identity-shortcut adds per slab, the resize of both 80-channel
    slabs to 128 x 128 whatever the input size, and the heads reading the two slabs."""
    from centerpose_b200.plan import (FLAG_CLIP01, OP_AVGPOOL, OP_CONV, OP_DWCONV, OP_RESIZE_BILINEAR, OP_SCALE_ADD,
                                      OP_UPSAMPLE_ADD)
    plan = _plan("ghostnet", "fp32", 1, 256, 320)
    ops = plan.pb.ops
    census = Counter(o.type for o in ops)
    assert plan.out_shape == (128, 128)
    assert census[OP_RESIZE_BILINEAR] == 2 and census[OP_AVGPOOL] == 14 and census[OP_SCALE_ADD] == 14
    assert census[OP_UPSAMPLE_ADD] == 20 and all(o.stride == 1 for o in ops if o.type == OP_UPSAMPLE_ADD)
    # cheap ops; the stride-2 dw of blocks 1 and 2 (two slabs each); the shortcut dw of six blocks, the first on the
    # single-slab stem output
    assert census[OP_DWCONV] == 32 + 2 * 2 + 1 + 5 * 2
    clip = [o for o in ops if o.flags & FLAG_CLIP01]
    assert len(clip) == 14 and all(o.type == OP_CONV and o.srcs[0].H == 1 for o in clip)
    resized = [o for o in ops if o.type == OP_RESIZE_BILINEAR]
    assert all((o.srcs[0].H, o.srcs[0].W, o.srcs[0].C, o.dst.H, o.dst.W) == (32, 40, 80, 128, 128) for o in resized)
    head0 = [o for o in ops if o.type == OP_CONV and o.k == (3, 3) and o.cout == 256]
    assert len(head0) == 6 and all([s.C for s in o.srcs] == [80, 80] for o in head0)
    assert all(s.C % 16 == 0 for o in ops for s in o.srcs if s.kind != "nchw_in")


@pytest.mark.parametrize("arch", sorted(ARCHS))
def test_split_plan_islands_at_512(arch):
    """fp16x2 at 512x512: every conv on a map of at least 8 columns is tensor-core eligible, ReLU6 / the deconv / the
    ghost slabs run natively on the planes, so the only CONVERT ops (fp32 islands) are around the SE's 1x1-map convs
    (GhostNet), as in the MobileNetV3 lowering; MobileNetV2 has none."""
    from centerpose_b200.plan import FLAG_TC, OP_CONV, OP_CONVERT
    plan = _plan(arch, "fp16x2", 1, 512, 512)
    ops = plan.pb.ops
    conv = [o for o in ops if o.type == OP_CONV]
    assert all(o.flags & FLAG_TC for o in conv if o.srcs[0].W >= 8)
    cvt = [o for o in ops if o.type == OP_CONVERT]
    if arch == "mobilenetv2":
        assert not cvt
    else:
        assert all(o.srcs[0].H == 1 and o.srcs[0].W == 1 for o in cvt)


@pytest.mark.parametrize("arch", sorted(ARCHS))
def test_checkpoint_roundtrip_reference_format(arch, tmp_path, capsys):
    """A reference-format checkpoint ({'epoch', 'state_dict'}, DataParallel 'module.' prefix) loads through load_model
    with no missing and no dropped keys."""
    from centerpose_b200.model import load_model, save_model
    from oracle.init_recipe import conditioned_state_dict
    m, _ = _model(arch)
    p = str(tmp_path / f"{arch}.pth")
    save_model(p, 3, m)
    sd = conditioned_state_dict(torch.load(p, weights_only=False)["state_dict"], 9)
    torch.save({"epoch": 3, "state_dict": {"module." + k: v for k, v in sd.items()}}, p)
    capsys.readouterr()
    m2 = load_model(_model(arch)[0], p)
    out = capsys.readouterr().out
    assert "No param" not in out and "Drop parameter" not in out and "Skip loading" not in out, out
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k

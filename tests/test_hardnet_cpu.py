"""CPU tests (-m "not gpu") of the HarDNet backbone (centerpose_b200/archs/hardnet.py): the oracle against the
reference-generated goldens, the parameter tree's key names / shapes / order, the lowering's op census and the
reference checkpoint format."""
import os
from collections import Counter

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _sha(*arrays):
    import hashlib
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _model():
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    cfg = default_cfg("hardnet")
    return create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg), cfg


@pytest.mark.parametrize("tag", ["128", "96x160"])
def test_hardnet_oracle_matches_reference_golden(tag):
    """oracle/hardnet_ref.py restates hardnet.py's forward; the goldens are the unmodified reference's own head maps."""
    from oracle import hardnet_ref
    from oracle.init_recipe import conditioned_state_dict, synth_images
    g = np.load(os.path.join(GOLD, f"hardnet_{tag}.npz"))
    B, H, W = [int(v) for v in g["shape"]]
    m, _ = _model()
    sd = conditioned_state_dict(m.state_dict(), 317)
    x = synth_images(B, H, W, 317)
    assert _sha(x.numpy()) == str(g["x_sha"])
    maps = torch.cat(hardnet_ref.forward(sd, x), dim=1).numpy()
    ref = g["maps"]
    assert maps.shape == ref.shape
    assert np.abs(maps - ref).max() <= 1e-4 * np.abs(ref).max()


def test_hardnet_state_dict_matches_reference():
    """438 entries (69 ConvLayers x (conv weight + 5 BatchNorm entries) + 24 head tensors); the conditioned weights'
    sha equals the golden's, which pins every key name and shape (the recipe draws in sorted-key order)."""
    from oracle.init_recipe import conditioned_state_dict
    m, _ = _model()
    own = m.state_dict()
    sd = conditioned_state_dict(own, 317)
    assert len(sd) == 438
    assert _sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()]) == str(np.load(os.path.join(GOLD, "hardnet_512.npz"))["sd_sha"])
    keys = list(own)
    assert keys[0] == "backbone_model.base.0.conv.weight" and keys[-1] == "head_model.hp_offset.2.bias"
    # the reference registers every denseBlocksUp before any conv1x1_up
    last_dense = max(i for i, k in enumerate(keys) if ".denseBlocksUp." in k)
    first_1x1 = min(i for i, k in enumerate(keys) if ".conv1x1_up." in k)
    assert last_dense < first_1x1
    assert own["backbone_model.base.16.layers.7.conv.weight"].shape[0] == 158    # 32 * 1.7^3 = 157.2, rounded to even
    assert own["backbone_model.conv1x1_up.0.conv.weight"].shape[:2] == (267, 534)
    bb = sum(v.numel() for k, v in own.items() if k.startswith("backbone_model.") and k.rsplit(".", 1)[1] in ("weight", "bias"))
    assert abs(bb / 1e6 - 4.12) < 0.01


def test_hardnet_link_rule():
    from centerpose_b200.archs import hardnet as hd
    assert [hd.links(l) for l in (1, 2, 3, 4, 6, 8)] == [[0], [1, 0], [2], [3, 2, 0], [5, 4], [7, 6, 4, 0]]
    assert hd.block_widths(48, 10, 4) == [48, 10, 18, 10, 28]
    assert hd.block_outputs(4) == [1, 3, 4] and hd.block_outputs(8) == [1, 3, 5, 7, 8]
    assert hd.block_widths(48, 16, 4)[4] == 46


def test_hardnet_plan_census():
    """fp32 lowering of the whole network on the CPU: every op reads at most four inputs, every input slab is a multiple
    of 16 channels, the heads run at stride 4, four 2x2 average pools and one resize per up-path slab (1 + 5 + 5 + 3)."""
    from centerpose_b200.plan import OP_AVGPOOL2, OP_CONV, OP_RESIZE_BILINEAR, OP_STEM
    m, _ = _model()
    m.set_precision("fp32")
    plan = m._plan(2, 128, 160, torch.device("cpu"))
    census = Counter(o.type for o in plan.ops)
    assert all(1 <= o.nsrc <= 4 for o in plan.ops)
    assert all(o.cin[j] % 16 == 0 for o in plan.ops if o.type != OP_STEM for j in range(o.nsrc))
    assert plan.out_shape == (32, 40)
    assert census[OP_AVGPOOL2] == 4
    assert census[OP_RESIZE_BILINEAR] == 14
    # 68 backbone ConvLayers after the stem + 8 extra chained chunk convs (three 5-slab 1x1s; up path 6, 10, 8, 6 slabs)
    # + 12 head convs
    assert census == {OP_STEM: 1, OP_CONV: 68 + 8 + 12, OP_AVGPOOL2: 4, OP_RESIZE_BILINEAR: 14}, census
    # the head's first 3x3 convs read the last up block's three slabs: 10 + 10 + 28 real channels in 16 + 16 + 32
    head0 = [o for o in plan.ops if o.type == OP_CONV and o.kh == 3 and o.cout == 256]
    assert len(head0) == 6 and all([o.cin[j] for j in range(o.nsrc)] == [16, 16, 32] for o in head0)
    pools = [o for o in plan.ops if o.type == OP_AVGPOOL2]
    assert all(o.Ho == o.H // 2 and o.Wo == o.W // 2 for o in pools)


def test_hardnet_split_plan_has_no_fp32_island_at_512():
    """fp16x2 at 512x512: the stride-2 stem takes the space-to-depth route, every conv is tensor-core eligible and the
    pool / resize ops run on the split planes, so the program holds no CONVERT op."""
    from centerpose_b200.plan import OP_CONV, OP_CONVERT
    m, _ = _model()
    m.set_precision("fp16x2")
    plan = m._plan(1, 512, 512, torch.device("cpu"))
    assert sum(o.type == OP_CONVERT for o in plan.ops) == 0
    assert all(o.flags & 8 for o in plan.ops if o.type == OP_CONV)


def test_hardnet_default_cfg_builds():
    m, cfg = _model()
    assert cfg.MODEL.HEAD_CONV == 256 and cfg.MODEL.INTERMEDIATE_CHANNEL == 48
    assert m.head_model.hm._modules["0"].weight.shape == (256, 48, 3, 3)


def test_hardnet_checkpoint_roundtrip_reference_format(tmp_path, capsys):
    """A reference-format checkpoint ({'epoch', 'state_dict'} with backbone_model.base.* keys, DataParallel 'module.'
    prefix) loads through load_model with no missing and no dropped keys."""
    from centerpose_b200.model import load_model, save_model
    from oracle.init_recipe import conditioned_state_dict
    m, cfg = _model()
    p = str(tmp_path / "hardnet.pth")
    save_model(p, 11, m)
    ck = torch.load(p, weights_only=False)
    assert set(ck) == {"epoch", "state_dict"} and "backbone_model.base.0.conv.weight" in ck["state_dict"]
    sd = conditioned_state_dict(ck["state_dict"], 5)
    torch.save({"epoch": 11, "state_dict": {"module." + k: v for k, v in sd.items()}}, p)
    capsys.readouterr()
    m2 = load_model(_model()[0], p)
    out = capsys.readouterr().out
    assert "No param" not in out and "Drop parameter" not in out and "Skip loading" not in out, out
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k

"""CPU tests of the validation pass (centerpose_b200/val.py): the numpy restatement (oracle/val_ref.py) against the
reference's targets and loss stats in tests/golden/val_targets.npz, the host table packing, and the refused settings."""
import math
import os
import types

import numpy as np
import pytest

from centerpose_b200.coco_eval import gt_table
from centerpose_b200.config import default_cfg
from centerpose_b200.image import get_affine_transform
from centerpose_b200 import val
from oracle import val_ref
from tests.val_cases import constructed, shapes_of

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = [n for n, _, _ in val.TARGETS]


def _restated(ds, R=128):
    out = {}
    for im in ds["images"]:
        c, s = val.center_scale(im["height"], im["width"])
        anns = [a for a in ds["annotations"] if a["image_id"] == im["id"]]
        out[im["id"]] = val_ref.targets(gt_table(anns), get_affine_transform(c, s, 0, [R, R]), R)
    return out


def test_restatement_equals_reference_targets():
    g = np.load(os.path.join(GOLD, "val_targets.npz"))
    ds = constructed()
    for image_id, tg in _restated(ds).items():
        for k in KEYS:
            want = g["%d/%s" % (image_id, k)]
            assert tg[k].dtype == want.dtype and tg[k].shape == want.shape, (image_id, k)
            assert np.array_equal(tg[k].view(np.uint8), want.view(np.uint8)), (image_id, k)


def test_golden_cases_reach_their_branches():
    g = np.load(os.path.join(GOLD, "val_targets.npz"))
    assert not g["2/reg_mask"].any() and not g["2/hm"].any()                   # all crowds: nothing kept
    assert g["3/ind"].shape == (32,) and g["3/reg_mask"].sum() > 0               # 39 non-crowd objects, 32 slots
    # image 1, slot 2: the zero-keypoint object: drawn, reg_mask 0, its centre raised from 0.9999 to 1.0
    assert g["1/reg_mask"][2] == 0 and g["1/wh"][2].all()
    assert g["1/hm"].reshape(-1)[g["1/ind"][2]] == 1.0
    # image 4: a box that clips to w = 0 and one that clips to h = 0 are not drawn
    assert not g["4/wh"][3].any() and not g["4/wh"][4].any()
    radii = {val_ref.radius(math.ceil(h), math.ceil(w)) for im in range(1, 9) for w, h in g["%d/wh" % im] if w > 0}
    assert 0 in radii and max(radii) >= 30
    for (h, w) in [(100, 347), (100, 503), (100, 685)]:
        c, s = val.center_scale(h, w)
        t = get_affine_transform(c, s, 0, [128, 128])
        assert t[0, 1] != 0 or t[1, 0] != 0


def test_restated_loss_within_2e6_of_reference():
    from oracle.make_golden_val import loss_logits
    g = np.load(os.path.join(GOLD, "val_targets.npz"))
    cfg = default_cfg("dla_34")
    ds = constructed()
    for im, seed, want in zip(ds["images"], g["loss_seeds"], g["loss_stats"]):
        tg = {k: g["%d/%s" % (im["id"], k)] for k in KEYS}
        got = val_ref.loss(loss_logits(int(seed)), tg, cfg.LOSS)
        assert np.all(np.abs(got - want) <= 2e-6 * np.abs(want)), (im["id"], got, want)


def test_radius_bound_at_output_128():
    r = [val_ref.radius(h, w) for h in range(1, 129) for w in range(1, 129)]
    assert min(r) == 0 and max(r) == 34


def test_image_table_packing():
    ds = constructed()
    ev = types.SimpleNamespace(gt_range={1: (0, 5), 4: (12, 7)}, cat_id=1)
    sh = shapes_of(ds)
    t = val.image_table(ev, [4, 1], [sh[4], sh[1]], 128)
    assert t.dtype.itemsize == 64 and t["gt_begin"].tolist() == [12, 0] and t["gt_count"].tolist() == [7, 5]
    c, s = val.center_scale(*sh[1])
    assert c.dtype == np.float32 and c.tolist() == [320.0, 240.0] and s == 640.0
    assert np.array_equal(t[1]["trans_output"], get_affine_transform(c, s, 0, [128, 128]).reshape(6))
    c, _ = val.center_scale(333, 517)
    assert c.tolist() == [258.5, 166.5]
    with pytest.raises(ValueError, match="not in the ground truth"):
        val.image_table(ev, [9], [(10, 10)], 128)
    with pytest.raises(ValueError, match="shapes"):
        val.image_table(ev, [1], [], 128)


@pytest.mark.parametrize("section, key, value", [
    ("LOSS", "MSE_LOSS", True), ("LOSS", "DENSE_HP", True), ("LOSS", "REG_LOSS", "sl1"),
    ("MODEL", "NUM_STACKS", 2), ("TEST", "EVAL_ORACLE_HM", True), ("TEST", "EVAL_ORACLE_HP_OFFSET", True),
    ("MODEL", "OUTPUT_RES", 64)])
def test_refused_settings(section, key, value):
    cfg = default_cfg("dla_34")
    val.check_cfg(cfg, types.SimpleNamespace(cat_id=1))
    cfg[section][key] = value
    with pytest.raises(NotImplementedError):
        val.check_cfg(cfg)


def test_refused_category_and_defaults():
    cfg = default_cfg("dla_34")
    with pytest.raises(NotImplementedError, match="category"):
        val.check_cfg(cfg, types.SimpleNamespace(cat_id=2))
    L = cfg.LOSS
    assert (L.HM_WEIGHT, L.WH_WEIGHT, L.OFF_WEIGHT, L.HP_WEIGHT, L.HM_HP_WEIGHT, L.REG_LOSS, L.DENSE_HP) == \
        (1., 0.1, 1., 1., 1., "l1", False) and cfg.MODEL.NUM_STACKS == 1

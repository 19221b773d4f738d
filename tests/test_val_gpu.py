"""GPU tests of the validation pass: the targets kernel (cpb200_multi_pose_targets_batch) bit for bit against the
reference's targets (tests/golden/val_targets.npz) and the numpy restatement (oracle/val_ref.py), the radius and every
Gaussian stamp exhaustively, the dataset normalisation (cpb200_pre_process_batch_f32) bit for bit, the loss kernel
against the reference's stats, and MultiPoseDetector.run_val end to end against tests/golden/val_dla34.npz."""
import ctypes
import math
import os

import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import _lib, val
from centerpose_b200.coco_eval import KeypointEval, gt_table
from centerpose_b200.config import default_cfg
from centerpose_b200.image import get_affine_transform
from oracle import val_ref
from tests.val_cases import _ann, _dataset, _person, constructed, random_case, shapes_of

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = [n for n, _, _ in val.TARGETS]


def _device_targets(ds, cfg=None):
    cfg = cfg or default_cfg("dla_34")
    ev = KeypointEval(ds)
    sh = shapes_of(ds)
    ids = [im["id"] for im in ds["images"]]
    tg = val.targets(ev, ids, [sh[i] for i in ids], cfg)
    return ids, {k: v.cpu().numpy() for k, v in tg.items()}


def _restated(ds, image_id, R=128):
    im = next(im for im in ds["images"] if im["id"] == image_id)
    c, s = val.center_scale(im["height"], im["width"])
    anns = [a for a in ds["annotations"] if a["image_id"] == image_id]
    return val_ref.targets(gt_table(anns), get_affine_transform(c, s, 0, [R, R]), R)


def _same(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    bad = np.flatnonzero(got.view(np.uint8) != want.view(np.uint8))
    assert bad.size == 0, (what, "%d differing bytes, the first at %d" % (bad.size, int(bad[0])))


def test_radius_exhaustive():
    hw = np.array([(h, w) for h in range(1, 129) for w in range(1, 129)], np.int32)
    d = torch.from_numpy(hw).cuda()
    out = torch.empty(len(hw), dtype=torch.int32, device="cuda")
    _lib.launch("gaussian_radius", d.device, d, len(hw), out)
    want = np.array([val_ref.radius(int(h), int(w)) for h, w in hw], np.int32)
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    assert want.max() == 34


def test_every_stamp_radius_0_to_34():
    """One object per 512x512 image, square boxes of 1..127 output pixels centred in the output: every radius 0..34
    is drawn whole, and the kernel's hm equals float32(gaussian2D) there bit for bit."""
    images, anns = [], []
    for n, side in enumerate(range(1, 128), start=1):
        x0 = 4 * (64 - side / 2)
        images.append((n, 512, 512))
        anns.append(_ann(n, n, [x0, x0, 4 * side, 4 * side], np.zeros((17, 3))))
    ds = _dataset(images, anns)
    ids, tg = _device_targets(ds)
    seen = set()
    for b, image_id in enumerate(ids):
        w, h = tg["wh"][b, 0]
        r = val_ref.radius(math.ceil(h), math.ceil(w))
        cx, cy = int(tg["ind"][b, 0] % 128), int(tg["ind"][b, 0] // 128)
        win = tg["hm"][b, 0, cy - r:cy + r + 1, cx - r:cx + r + 1]
        _same(win, val_ref.stamp(r), ("stamp", r))
        _same(tg["hm"][b], _restated(ds, image_id)["hm"], ("hm", image_id))
        seen.add(r)
    assert seen == set(range(35))


def test_targets_equal_reference_golden():
    g = np.load(os.path.join(GOLD, "val_targets.npz"))
    ids, tg = _device_targets(constructed())
    for b, image_id in enumerate(ids):
        for k in KEYS:
            _same(tg[k][b], g["%d/%s" % (image_id, k)], (image_id, k))


def test_zero_keypoint_object_centre():
    """hm[ct] = 0.9999 for an object without keypoints, then its own stamp: 1.0 there, reg_mask 0, its wh and ind
    set; a later object's stamp over that centre does not lower it."""
    rng = np.random.default_rng(3)
    anns = [_ann(1, 1, [100, 100, 80, 160], np.zeros((17, 3))),
            _ann(2, 1, [90, 90, 120, 200], _person(rng, 90, 90, 120, 200))]
    ds = _dataset([(1, 400, 400)], anns)
    _, tg = _device_targets(ds)
    assert tg["reg_mask"][0].tolist()[:2] == [0, 1]
    assert tg["hm"][0].reshape(-1)[tg["ind"][0, 0]] == 1.0
    for k in KEYS:
        _same(tg[k][0], _restated(ds, 1)[k], k)


def test_targets_equal_restatement_on_300_seeded_sets():
    for seed in range(300):
        ds = random_case(seed, n_images=2)
        ids, tg = _device_targets(ds)
        for b, image_id in enumerate(ids):
            want = _restated(ds, image_id)
            for k in KEYS:
                _same(tg[k][b], want[k], (seed, image_id, k))


def test_pre_process_f32_equals_dataset_normalisation():
    from centerpose_b200.detector import pack_group
    cfg = default_cfg("dla_34")
    res = 512
    rng = np.random.RandomState(9)
    shapes = [(480, 640), (641, 427), (333, 517), (512, 512), (37, 1001)]
    images = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in shapes]
    trans = [get_affine_transform(*val.center_scale(h, w), 0, [res, res]) for h, w in shapes]
    host, at = pack_group(images, shapes, trans, np.zeros((len(images), 6), np.float32), list(range(len(images))))
    buf = torch.from_numpy(host).cuda()
    out = torch.empty((len(images), 3, res, res), dtype=torch.float32, device="cuda")
    mean = (ctypes.c_float * 3)(*np.float32(cfg.DATASET.MEAN))
    std = (ctypes.c_float * 3)(*np.float32(cfg.DATASET.STD))
    _lib.launch("pre_process_batch_f32", out.device, buf.data_ptr() + at["o_img"], buf, len(images), out, res, res, mean,
                std)
    got = out.cpu().numpy()
    for n, (im, t) in enumerate(zip(images, trans)):
        want = np.ascontiguousarray(val_ref.inputs(im, t, res, cfg.DATASET.MEAN, cfg.DATASET.STD))
        _same(got[n], want, ("input", shapes[n]))


def test_loss_kernel_against_reference_stats():
    from oracle.make_golden_val import loss_logits
    g = np.load(os.path.join(GOLD, "val_targets.npz"))
    cfg = default_cfg("dla_34")
    ds = constructed()
    ids = [im["id"] for im in ds["images"]]
    heads = [loss_logits(int(s)) for s in g["loss_seeds"]]
    outputs = [torch.from_numpy(np.stack([h[c] for h in heads])).cuda() for c in range(6)]
    tg = {k: torch.from_numpy(np.stack([g["%d/%s" % (i, k)] for i in ids])).cuda() for k in KEYS}
    got = val.loss(outputs, tg, cfg).cpu().numpy()
    want = g["loss_stats"]
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-30)
    assert np.all((got == want) | (rel <= 1e-5)), (rel.max(), got, want)
    for b, i in enumerate(ids):
        mine = val_ref.loss(heads[b], {k: g["%d/%s" % (i, k)] for k in KEYS}, cfg.LOSS)
        ulp = np.abs(got[b].view(np.int32).astype(np.int64) - mine.view(np.int32).astype(np.int64))
        assert ulp.max() <= 2, (i, got[b], mine)
    # the logits are read, not modified
    assert torch.equal(outputs[0].cpu(), torch.from_numpy(np.stack([h[0] for h in heads])))


# measured on an H100: at most 3e-6 relative in fp32 and 2.4e-5 in fp16x2
@pytest.mark.parametrize("precision, tol", [("fp32", 1e-5), ("fp16x2", 1e-4)])
def test_run_val_matches_reference_val_pass(precision, tol, tmp_path):
    from centerpose_b200.detector import detector_factory
    from oracle import make_golden_val as g
    from oracle.init_recipe import conditioned_state_dict
    from tests.util import match_rows
    f = np.load(os.path.join(GOLD, "val_dla34.npz"))
    pixels = [g.image(seed, h, w) for seed, h, w in g.VAL_IMAGES]
    assert str(f["img_sha"]) == g._sha(*pixels)
    paths = []
    for (seed, _, _), px in zip(g.VAL_IMAGES, pixels):
        paths.append(str(tmp_path / ("%d.png" % seed)))
        cv2.imwrite(paths[-1], px)
    cfg = default_cfg("dla_34")
    cfg.B200.PRECISION = precision
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    ev = KeypointEval(g.dla34_case())
    ids = f["image_ids"].tolist()
    assert ev.cat_img_ids == sorted(ids)
    log, preds = det.run_val(paths, ids, ev, max_batch=2)
    got = np.array([log[k] for k in val.STATS])
    rel = np.abs(got - f["stats"]) / np.abs(f["stats"])
    print(precision, "run_val stats relative error", dict(zip(val.STATS, rel.round(8).tolist())))
    assert rel.max() <= tol, (precision, rel)
    assert log["time"] > 0 and set(preds) == set(ids)
    for i in ids:
        rows = preds[i][1]
        want = f["preds_%d" % i]
        assert rows.dtype == np.float32 and rows.shape == want.shape
        m_rows, m_elems = match_rows(rows, want, tol=1e-3, box_tol=5e-2)
        print(precision, "image", i, "rows matched", round(m_rows, 4), "elements", round(m_elems, 4))
        assert m_rows >= 0.9 and m_elems >= 0.97, (precision, i, m_rows, m_elems)
    stats = ev.evaluate(preds)
    assert len(stats) == 10
    # arrays take the same path as files
    log2, preds2 = det.run_val(pixels, ids, ev, max_batch=2)
    assert all(log2[k] == log[k] for k in val.STATS)
    assert all(np.array_equal(preds2[i][1], preds[i][1]) for i in ids)


def test_run_val_refusals():
    from centerpose_b200.detector import detector_factory
    from oracle import make_golden_val as g
    cfg = default_cfg("dla_34")
    det = detector_factory[cfg.TEST.TASK](cfg)
    ev = KeypointEval(g.dla34_case())
    px = [g.image(1, 64, 64)]
    with pytest.raises(ValueError, match="not in the ground truth"):
        det.run_val(px, [999], ev)
    with pytest.raises(ValueError, match="image ids"):
        det.run_val(px, [], ev)
    det.cfg.LOSS.MSE_LOSS = True
    with pytest.raises(NotImplementedError):
        det.run_val(px, [301], ev)

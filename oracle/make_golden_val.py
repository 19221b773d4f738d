"""Generate ``tests/golden/val_targets.npz`` and ``tests/golden/val_dla34.npz`` from the UNMODIFIED reference's
validation pass on the CPU, and pin the numpy restatement (``oracle/val_ref.py``) against it before anything is
written.

Run:  python -m oracle.make_golden_val      (from the repo root; needs /root/reference)

How the reference runs:
  * ``MultiPoseDataset.__getitem__`` (lib/datasets/multi_pose.py) on an object made with ``object.__new__``, split
    'val', with a stub ``coco`` (``loadImgs`` / ``getAnnIds`` / ``loadAnns`` over the case's dict, annotations per
    image in file order as pycocotools indexes them).  Its ``annToMask`` returns zeros: ``segment`` reaches no returned
    target, and pycocotools is not installed.  ``utils.image`` is ``ref_harness``'s patched module.
  * ``MultiPoseLoss.forward``, ``MultiPoseTrainer.save_result`` (lib/trains/multi_pose.py) and ``AverageMeter``
    (lib/utils/utils.py) on the collated batch of one image, as ``BaseTrainer.run_epoch('val')`` calls them.
    ``progress.bar`` is stubbed.

val_targets.npz: per image ``<image id>/<key>`` for the eleven targets of ``tests/val_cases.constructed()``, and for the
loss test ``loss_seeds`` (one seed per image: the six head maps are ``loss_logits(seed)``) and ``loss_stats``
((images, 7), the reference's float32 stats).
val_dla34.npz: DLA-34 with ``conditioned_state_dict(..., 317)`` on ``VAL_IMAGES`` (seeded images, written as PNG and
read back by ``cv2.imread``; ``img_sha`` of the pixels), ground truth ``dla34_case()``: ``stats`` (the seven
averaged stats in ``val_ref.STATS`` order), ``preds_<image id>`` (the (100, 56) rows of ``save_result``),
``image_ids``, ``sd_sha``.
"""
from __future__ import annotations

import hashlib
import os
import sys
import tempfile
import types

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
OUT_TARGETS = os.path.join(GOLD, "val_targets.npz")
OUT_DLA = os.path.join(GOLD, "val_dla34.npz")

KEYS = ["hm", "hm_hp", "wh", "reg", "ind", "reg_mask", "hps", "hps_mask", "hp_offset", "hp_ind", "hp_mask"]
VAL_IMAGES = [(301, 240, 320), (302, 300, 200), (303, 333, 517)]       # (seed, h, w)
HEAD_CHANNELS = (1, 2, 34, 2, 17, 2)


def image(seed, h, w):
    """A seeded BGR image: smooth blobs over noise, so the network's maps have structure."""
    rng = np.random.RandomState(seed)
    img = rng.randint(0, 256, size=(h // 8 + 1, w // 8 + 1, 3)).astype(np.uint8)
    img = cv2.resize(img, (w, h), interpolation=cv2.INTER_CUBIC)
    return np.clip(img.astype(np.int16) + rng.randint(-20, 21, size=(h, w, 3)), 0, 255).astype(np.uint8)


def loss_logits(seed, R=128):
    """The six seeded (C, R, R) float32 head maps of the loss test: logits for hm and hm_hp around -3, whose
    sigmoid spans the clamp bounds, and regression maps of the targets' scale."""
    rng = np.random.RandomState(seed)
    out = []
    for n, c in enumerate(HEAD_CHANNELS):
        if n in (0, 4):
            out.append((rng.standard_normal((c, R, R)) * 3 - 3).astype(np.float32))
        else:
            out.append((rng.standard_normal((c, R, R)) * (10 if n in (1, 2) else 0.5)).astype(np.float32))
    return out


def dla34_case():
    """The ground truth of ``VAL_IMAGES``: a few people per image, a crowd and a zero-keypoint one among them."""
    from tests.val_cases import _ann, _dataset, _person
    rng = np.random.default_rng(11)
    anns, aid = [], 1
    for n, (seed, h, w) in enumerate(VAL_IMAGES):
        for k in range(4):
            bw, bh = rng.uniform(0.2, 0.6) * w, rng.uniform(0.3, 0.9) * h
            x, y = rng.uniform(0, w - bw), rng.uniform(0, h - bh)
            vis = "none" if (n, k) == (1, 2) else "partial"
            anns.append(_ann(aid, seed, [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)],
                             _person(rng, x, y, bw, bh, vis), crowd=int((n, k) == (0, 3))))
            aid += 1
    return _dataset([(seed, h, w) for seed, h, w in VAL_IMAGES], anns)


def _sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def ref_cfg():
    """The reference cfg the dataset and the loss read: the package defaults plus TEST.EVAL_ORACLE_* off."""
    from centerpose_b200.config import default_cfg
    from oracle.ref_harness import AttrDict
    cfg = AttrDict(default_cfg("dla_34"))
    for k in ("HM", "WH", "OFFSET", "KPS", "HMHP", "HP_OFFSET", "DEP"):
        cfg.TEST["EVAL_ORACLE_" + k] = False
    return cfg


def _reference():
    from oracle.ref_harness import load_reference
    load_reference()
    if "progress.bar" not in sys.modules:
        progress = types.ModuleType("progress"); bar = types.ModuleType("progress.bar")
        bar.Bar = object; progress.bar = bar
        sys.modules["progress"] = progress; sys.modules["progress.bar"] = bar
    import importlib.util
    from oracle.ref_harness import REF_ROOT
    # an installed package may own the name `datasets`; the reference's module is loaded from its file
    path = os.path.join(REF_ROOT, "lib", "datasets", "multi_pose.py")
    spec = importlib.util.spec_from_file_location("ref_datasets_multi_pose", path)
    ref_ds = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref_ds)
    import trains.multi_pose as ref_tr
    import utils.utils as ref_utils
    return ref_ds, ref_tr, ref_utils


class _Coco:
    """The slice of pycocotools' COCO that __getitem__ calls."""

    def __init__(self, ds):
        self.imgs = {im["id"]: im for im in ds["images"]}
        self.anns = {a["id"]: a for a in ds["annotations"]}
        self.img_to_anns = {i: [] for i in self.imgs}
        for a in ds["annotations"]:
            self.img_to_anns[a["image_id"]].append(a["id"])

    def loadImgs(self, ids):
        return [self.imgs[i] for i in ids]

    def getAnnIds(self, imgIds):
        return [a for i in imgIds for a in self.img_to_anns[i]]

    def loadAnns(self, ids):
        return [self.anns[i] for i in ids]

    def annToMask(self, ann):
        im = self.imgs[ann["image_id"]]
        return np.zeros((im["height"], im["width"]), np.uint8)


def reference_items(ds, pixels, cfg):
    """``__getitem__`` of every image of ``ds`` (split 'val'); ``pixels[image id]`` is written as PNG first."""
    ref_ds, _, _ = _reference()
    with tempfile.TemporaryDirectory() as d:
        for im in ds["images"]:
            cv2.imwrite(os.path.join(d, im["file_name"]), pixels[im["id"]])
        dset = object.__new__(ref_ds.MultiPoseDataset)
        dset.images = [im["id"] for im in ds["images"]]
        dset.coco, dset.img_dir, dset.split, dset.cfg = _Coco(ds), d, "val", cfg
        dset._valid_ids, dset.max_objs, dset.num_joints, dset.num_classes = [1], 32, 17, 1
        dset.flip_idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
        return [dset.__getitem__(n) for n in range(len(dset.images))]


def restated(ds, pixels, cfg):
    """The restatement's targets and input of every image of ``ds``."""
    from centerpose_b200.coco_eval import gt_table
    from centerpose_b200.image import get_affine_transform
    from centerpose_b200.val import center_scale
    from oracle import val_ref
    per = {im["id"]: [a for a in ds["annotations"] if a["image_id"] == im["id"]] for im in ds["images"]}
    R, res = cfg.MODEL.OUTPUT_RES, cfg.MODEL.INPUT_RES
    out = []
    for im in ds["images"]:
        c, s = center_scale(im["height"], im["width"])
        tg = val_ref.targets(gt_table(per[im["id"]]), get_affine_transform(c, s, 0, [R, R]), R)
        tg["input"] = val_ref.inputs(pixels[im["id"]], get_affine_transform(c, s, 0, [res, res]), res,
                                     cfg.DATASET.MEAN, cfg.DATASET.STD)
        out.append(tg)
    return out


def pin_targets(ds, cfg, seed):
    """Asserts the restatement equals __getitem__ bit for bit on ``ds``; returns the reference's items."""
    pixels = {im["id"]: image(seed + im["id"], im["height"], im["width"]) for im in ds["images"]}
    ref = reference_items(ds, pixels, cfg)
    mine = restated(ds, pixels, cfg)
    for im, r, m in zip(ds["images"], ref, mine):
        for k in KEYS + ["input"]:
            a, b = np.ascontiguousarray(r[k]), np.ascontiguousarray(m[k])
            assert a.dtype == b.dtype and a.shape == b.shape, (im["id"], k, a.dtype, b.dtype, a.shape, b.shape)
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), ("restatement != __getitem__", im["id"], k)
    return ref


def _batch(item):
    return {k: torch.from_numpy(np.asarray(item[k]))[None] for k in KEYS}


def reference_loss(ref_tr, cfg, heads, item):
    """MultiPoseLoss.forward on one image: the seven stats as ``loss_stats[l].mean().item()``."""
    crit = ref_tr.MultiPoseLoss(cfg, 0)
    _, st = crit([torch.from_numpy(np.ascontiguousarray(h))[None].clone() for h in heads], _batch(item))
    return np.array([st[k].mean().item() for k in ("loss", "hm_loss", "hp_loss", "hm_hp_loss", "hp_offset_loss",
                                                   "wh_loss", "off_loss")], np.float32)


def main():
    from oracle import val_ref
    from oracle.make_golden_run import state_dict
    from tests.val_cases import constructed, random_case
    cfg = ref_cfg()
    _, ref_tr, ref_utils = _reference()

    # targets: the constructed cases stored, seeded cases pinned
    ds = constructed()
    ref = pin_targets(ds, cfg, 400)
    for seed in range(40):
        pin_targets(random_case(seed), cfg, 500 + 10 * seed)
    print("restatement == __getitem__ on the constructed cases and 40 seeded ones")
    out = {}
    for im, r in zip(ds["images"], ref):
        for k in KEYS:
            out["%d/%s" % (im["id"], k)] = np.asarray(r[k])
    seeds = np.array([700 + im["id"] for im in ds["images"]])
    stats = []
    for s, r in zip(seeds, ref):
        heads = loss_logits(int(s))
        want = reference_loss(ref_tr, cfg, heads, r)
        got = val_ref.loss(heads, r, cfg.LOSS)
        assert np.all(np.abs(got - want) <= 2e-6 * np.abs(want)), ("restated loss", s, got, want)
        stats.append(want)
    out["loss_seeds"], out["loss_stats"] = seeds, np.stack(stats)
    np.savez_compressed(OUT_TARGETS, **out)
    print("wrote", OUT_TARGETS, os.path.getsize(OUT_TARGETS), "bytes")

    # DLA-34 through the reference's val loop
    from oracle.ref_harness import ref_create_model
    sd = state_dict()
    model, _ = ref_create_model("dla_34_512x512")
    model.load_state_dict(sd)
    ds = dla34_case()
    pixels = {seed: image(seed, h, w) for seed, h, w in VAL_IMAGES}
    items = reference_items(ds, pixels, cfg)
    trainer = object.__new__(ref_tr.MultiPoseTrainer)
    trainer.cfg = cfg
    crit = ref_tr.MultiPoseLoss(cfg, 0)
    meters = {k: ref_utils.AverageMeter() for k in val_ref.STATS}
    results = {}
    with torch.no_grad():
        for item in items:
            batch = _batch(item)
            batch["input"] = torch.from_numpy(item["input"])[None]
            batch["meta"] = {"c": torch.from_numpy(item["meta"]["c"])[None],
                             "s": torch.tensor([item["meta"]["s"]]), "img_id": torch.tensor([item["meta"]["img_id"]])}
            outputs = model(batch["input"])
            _, st = crit(outputs, batch)
            for k in meters:
                meters[k].update(st[k].mean().item(), 1)
            trainer.save_result(outputs, batch, results)
    out = {"image_ids": np.array([seed for seed, _, _ in VAL_IMAGES]),
           "shapes": np.array([[h, w] for _, h, w in VAL_IMAGES]),
           "stats": np.array([meters[k].avg for k in val_ref.STATS], np.float64),
           "sd_sha": np.array(_sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])),
           "img_sha": np.array(_sha(*[pixels[s] for s, _, _ in VAL_IMAGES]))}
    for i, r in results.items():
        out["preds_%d" % int(i)] = np.asarray(r[1], np.float32)
    print("stats", dict(zip(val_ref.STATS, out["stats"].tolist())))
    np.savez_compressed(OUT_DLA, **out)
    print("wrote", OUT_DLA, os.path.getsize(OUT_DLA), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()

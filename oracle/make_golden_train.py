"""Generate ``tests/golden/train_batches.npz`` from the UNMODIFIED reference's ``MultiPoseDataset.__getitem__`` for split
'train' on the CPU, and pin the host draws (``centerpose_b200.train_data.TrainDraws``) and the numpy restatement
(``oracle/train_ref.py``) against it before anything is written.

Run:  python -m oracle.make_golden_train      (from the repo root; needs /root/reference)

How the reference runs: as in ``make_golden_val.py`` (an object made with ``object.__new__``, the stub ``coco``, the
images written as PNG), with split 'train', ``_data_rng = RandomState(123)`` and COCOHP's ``_eig_val`` / ``_eig_vec``,
after ``np.random.seed`` and ``random.seed`` with the case's seeds.  What it drew is recorded without changing what it
does: ``get_affine_transform`` and ``cv2.warpAffine`` are wrapped in the module's namespace (the centre, scale and
rotation of the input matrix; whether the image was mirrored), and ``color_aug`` is wrapped to save the states of
``random`` and ``data_rng`` before the call, from which the shuffle, the alphas and ``np.dot``'s lighting vector are
replayed.

train_batches.npz, per case ``<case>/<image index>/<key>``: the sparse targets in full (``wh``, ``reg``, ``ind``,
``reg_mask``, ``hps``, ``hps_mask``, ``hp_offset``, ``hp_ind``, ``hp_mask``), SHA-256 of ``input``, ``hm`` and
``hm_hp`` (``<key>_sha``), and the draws: ``c``, ``s``, ``rot``, ``flip``, and with colour ``order``, ``alpha``,
``light``.  ``<case>/img_sha`` hashes the seeded pixels (``make_golden_val.image(1000 * case index + image id, h, w)``).
"""
from __future__ import annotations

import hashlib
import os
import random
import sys
import tempfile

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "train_batches.npz")

SPARSE = ["wh", "reg", "ind", "reg_mask", "hps", "hps_mask", "hp_offset", "hp_ind", "hp_mask"]
DENSE = ["input", "hm", "hm_hp"]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pixels(case_index, ds):
    from oracle.make_golden_val import image
    return {im["id"]: image(1000 * case_index + im["id"], im["height"], im["width"]) for im in ds["images"]}


class _Cv2:
    """cv2 as the dataset module sees it, with warpAffine noting whether its source is mirrored."""

    def __init__(self, log):
        self.log = log

    def __getattr__(self, name):
        return getattr(cv2, name)

    def warpAffine(self, img, *a, **k):
        self.log.append(img.strides[1] < 0)
        return cv2.warpAffine(img, *a, **k)


def reference_items(ds, pix, cfg, np_seed, py_seed):
    """The reference's ``__getitem__`` of every image of ``ds`` in order, and the draws each made."""
    from oracle.make_golden_val import _Coco, _reference
    ref_ds, _, _ = _reference()
    import utils.image as ref_image
    calls, flips, colors = [], [], []
    orig = (ref_ds.get_affine_transform, ref_ds.cv2, ref_ds.color_aug)

    def gat(c, s, rot, size, *a, **k):
        calls.append((np.array(c, np.float32), s, rot))
        return ref_image.get_affine_transform(c, s, rot, size, *a, **k)

    def aug(data_rng, image, eig_val, eig_vec):
        colors.append((random.getstate(), data_rng.get_state()))
        return ref_image.color_aug(data_rng, image, eig_val, eig_vec)

    ref_ds.get_affine_transform, ref_ds.cv2, ref_ds.color_aug = gat, _Cv2(flips), aug
    try:
        with tempfile.TemporaryDirectory() as d:
            for im in ds["images"]:
                cv2.imwrite(os.path.join(d, im["file_name"]), pix[im["id"]])
            dset = object.__new__(ref_ds.MultiPoseDataset)
            dset.images = [im["id"] for im in ds["images"]]
            dset.coco, dset.img_dir, dset.split, dset.cfg = _Coco(ds), d, "train", cfg
            dset._valid_ids, dset.max_objs, dset.num_joints, dset.num_classes = [1], 32, 17, 1
            dset.flip_idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
            dset._data_rng = np.random.RandomState(123)
            dset._eig_val = np.array([0.2141788, 0.01817699, 0.00341571], dtype=np.float32)
            dset._eig_vec = np.array([[-0.58752847, -0.69563484, 0.41340352], [-0.5832747, 0.00994535, -0.81221408],
                                      [-0.56089297, 0.71832671, 0.41158938]], dtype=np.float32)
            np.random.seed(np_seed)
            random.seed(py_seed)
            items = []
            for n in range(len(dset.images)):
                before, first, warp = len(colors), len(calls), len(flips)
                item = dset.__getitem__(n)
                c, s, rot = calls[first]               # the item's first matrix and warp are the input's
                draw = {"c": c, "s": s, "rot": rot, "flip": flips[warp], "color": len(colors) > before}
                if draw["color"]:
                    rs, ds_state = colors[-1]
                    r = random.Random()
                    r.setstate(rs)
                    order = [0, 1, 2]
                    r.shuffle(order)
                    g = np.random.RandomState()
                    g.set_state(ds_state)
                    draw["order"] = order
                    draw["alpha"] = [1. + g.uniform(low=-0.4, high=0.4) for _ in order]
                    draw["light"] = np.dot(dset._eig_vec, dset._eig_val * g.normal(scale=0.1, size=(3,)))
                items.append((item, draw))
            return items
    finally:
        ref_ds.get_affine_transform, ref_ds.cv2, ref_ds.color_aug = orig


def restated(ds, pix, cfg, np_seed, py_seed):
    """The host draws and the restatement's input and targets of every image of ``ds`` in order."""
    from centerpose_b200.coco_eval import gt_table
    from centerpose_b200.image import get_affine_transform
    from centerpose_b200.train_data import TrainDraws
    from oracle import train_ref
    per = {im["id"]: [a for a in ds["annotations"] if a["image_id"] == im["id"]] for im in ds["images"]}
    S, R = cfg.MODEL.INPUT_RES, cfg.MODEL.OUTPUT_RES
    draws = TrainDraws(cfg)
    np.random.seed(np_seed)
    random.seed(py_seed)
    out = []
    for im in ds["images"]:
        h, w = im["height"], im["width"]
        p = draws.draw(h, w)
        p["trans_input"] = get_affine_transform(p["c"], p["s"], p["rot"], [S, S])
        tg = train_ref.targets(gt_table(per[im["id"]]), w, p["flip"], p["rot"],
                               get_affine_transform(p["c"], p["s"], 0, [R, R]),
                               get_affine_transform(p["c"], p["s"], p["rot"], [R, R]), R)
        tg["input"] = train_ref.inputs(pix[im["id"]], p, S, cfg.DATASET.MEAN, cfg.DATASET.STD)
        out.append((tg, p))
    return out


def same_draw(a, b):
    if not (np.array_equal(a["c"].view(np.uint32), b["c"].view(np.uint32)) and float(a["s"]) == float(b["s"])
            and float(a["rot"]) == float(b["rot"]) and bool(a["flip"]) == bool(b["flip"])
            and a["color"] == b["color"]):
        return False
    if a["color"]:
        return (list(a["order"]) == list(b["order"]) and list(a["alpha"]) == list(b["alpha"])
                and np.array_equal(np.asarray(a["light"]), np.asarray(b["light"])))
    return True


def ref_cfg():
    from oracle.make_golden_val import ref_cfg as val_cfg
    cfg = val_cfg()
    cfg.DATASET.update({"RANDOM_CROP": True, "SHIFT": 0.1, "SCALE": 0.4, "ROTATE": 0., "AUG_ROT": 0., "FLIP": 0.5,
                        "NO_COLOR_AUG": False})
    return cfg


def main():
    from tests.train_cases import CASES, case_cfg, dataset
    base = ref_cfg()
    out = {}
    for ci, (name, settings, res, np_seed, py_seed) in enumerate(CASES):
        cfg = case_cfg(base, settings, res)
        ds = dataset(name)
        pix = pixels(ci, ds)
        ref = reference_items(ds, pix, cfg, np_seed, py_seed)
        mine = restated(ds, pix, cfg, np_seed, py_seed)
        assert len(ref) == len(mine)
        n_rot = n_flip = 0
        for n, ((item, rd), (tg, p)) in enumerate(zip(ref, mine)):
            assert same_draw(rd, p), ("host draws != the reference's", name, n, rd, p)
            for k in SPARSE + DENSE:
                a, b = np.ascontiguousarray(item[k]), np.ascontiguousarray(tg[k])
                assert a.dtype == b.dtype and a.shape == b.shape, (name, n, k, a.dtype, b.dtype, a.shape, b.shape)
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), ("restatement != __getitem__", name, n, k)
            for k in SPARSE:
                out["%s/%d/%s" % (name, n, k)] = np.asarray(item[k])
            for k in DENSE:
                out["%s/%d/%s_sha" % (name, n, k)] = np.array(sha(item[k]))
            for k in ("c", "s", "rot", "flip", "color"):
                out["%s/%d/%s" % (name, n, k)] = np.asarray(rd[k])
            if rd["color"]:
                for k in ("order", "alpha", "light"):
                    out["%s/%d/%s" % (name, n, k)] = np.asarray(rd[k])
            n_rot += rd["rot"] != 0
            n_flip += bool(rd["flip"])
        out["%s/img_sha" % name] = np.array(sha(np.concatenate([pix[im["id"]].reshape(-1) for im in ds["images"]])))
        print("%-20s %2d images, %d rotated, %d flipped: restatement == __getitem__" % (name, len(ref), n_rot, n_flip))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()

"""Cases of the training batches (``centerpose_b200.train_data``), shared by ``oracle/make_golden_train.py`` and the
tests: each is a dataset, the DATASET settings, the input resolution and the seeds of ``np.random`` and ``random``."""
import copy

import numpy as np

from tests.val_cases import J, _ann, _dataset, _person, constructed


def seeded_case(seed, n_images, lo=40, hi=700, people=(0, 41)):
    """A seeded dataset: images of random size in [lo, hi), random people around and across them, crowds, hidden and
    zero-keypoint people, joints anywhere."""
    rng = np.random.default_rng(3000 + seed)
    images, anns, aid = [], [], 1
    for i in range(n_images):
        h, w = int(rng.integers(lo, hi)), int(rng.integers(lo, hi))
        images.append((i + 1, h, w))
        for _ in range(int(rng.integers(*people))):
            bw, bh = rng.uniform(0.05, 0.8) * w, rng.uniform(0.05, 0.9) * h
            x, y = rng.uniform(-0.2 * w, w), rng.uniform(-0.2 * h, h)
            kps = _person(rng, x, y, bw, bh, rng.choice(["full", "partial", "partial", "none"]))
            if rng.random() < 0.2:
                kps[:, 0:2] = np.round(rng.uniform(-50, max(h, w) + 50, (J, 2)), 2)
            anns.append(_ann(aid, i + 1, [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)], kps,
                             crowd=int(rng.random() < 0.1)))
            aid += 1
    return _dataset(images, anns)


def small_case():
    """Images under 256 pixels a side (the crop border halves), one with more than 32 people."""
    rng = np.random.default_rng(41)
    images = [(1, 120, 200), (2, 250, 90), (3, 64, 64), (4, 200, 255)]
    anns, aid = [], 1
    for image_id, h, w in images:
        for n in range(40 if image_id == 1 else 3):
            bw, bh = rng.uniform(5, w / 2), rng.uniform(5, h / 2)
            x, y = rng.uniform(0, w - bw), rng.uniform(0, h - bh)
            anns.append(_ann(aid, image_id, [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)],
                             _person(rng, x, y, bw, bh, "none" if n == 2 else "partial"), crowd=int(n == 4)))
            aid += 1
    return _dataset(images, anns)


# name, DATASET settings, INPUT_RES, np.random seed, random seed
CASES = [
    ("crop", {}, 128, 1, 11),
    ("shift_rot", {"RANDOM_CROP": False, "AUG_ROT": 1., "ROTATE": 30.}, 128, 2, 12),
    ("crop_rot_nocolor", {"AUG_ROT": 0.5, "ROTATE": 30., "NO_COLOR_AUG": True}, 128, 3, 13),
    ("shift_flip_nocolor", {"RANDOM_CROP": False, "FLIP": 1., "NO_COLOR_AUG": True}, 128, 4, 14),
    ("small_flip", {"FLIP": 1.}, 128, 5, 15),
    ("seeded_rot", {"AUG_ROT": 0.5, "ROTATE": 30.}, 128, 6, 16),
    ("s512", {"AUG_ROT": 0.5, "ROTATE": 30.}, 512, 7, 17),
]


def dataset(name):
    if name in ("crop", "shift_rot", "crop_rot_nocolor", "shift_flip_nocolor"):
        return constructed()
    if name == "small_flip":
        return small_case()
    if name == "seeded_rot":
        return seeded_case(0, 8)
    return seeded_case(1, 2, lo=300, hi=700, people=(3, 8))


def seeded_jpeg_batch(tmp_path, B=32, res=512, seed=0, settings=None):
    """``(cfg, batch)``: a TrainData batch on the device from B seeded JPEG files written under ``tmp_path`` (images of
    200 to 700 pixels a side, 1 to 11 people each), at input resolution ``res``, with DLA-34's config and the DATASET
    ``settings`` (default: rotation and flips)."""
    import random

    import cv2

    from centerpose_b200 import train_data
    from centerpose_b200.config import default_cfg
    from oracle.make_golden_val import image
    cfg = case_cfg(default_cfg("dla_34"), settings or {"AUG_ROT": 0.3, "ROTATE": 30., "FLIP": 0.5}, res)
    ds = seeded_case(700 + seed, B, lo=200, hi=700, people=(1, 12))
    paths = []
    for im in ds["images"]:
        p = str(tmp_path / ("%d_%d.jpg" % (seed, im["id"])))
        cv2.imwrite(p, image(9000 + 100 * seed + im["id"], im["height"], im["width"]), [cv2.IMWRITE_JPEG_QUALITY, 90])
        paths.append(p)
    np.random.seed(60 + seed)
    random.seed(70 + seed)
    batch = train_data.TrainData(cfg, ds).batch(paths, [im["id"] for im in ds["images"]])
    return cfg, batch


def case_cfg(base, settings, res):
    """``base`` with the DATASET ``settings`` and the input resolution ``res`` (output res / 4)."""
    cfg = copy.deepcopy(base)
    for k, v in settings.items():
        cfg.DATASET[k] = v
    cfg.MODEL.INPUT_RES, cfg.MODEL.OUTPUT_RES = res, res // 4
    cfg.MODEL.INPUT_H = cfg.MODEL.INPUT_W = res
    return cfg

"""GPU tests of the training batches: TrainData.batch (cpb200_train_augment_batch and
cpb200_multi_pose_targets_train_batch) bit for bit against the reference's __getitem__ (tests/golden/train_batches.npz)
and against the numpy restatement (oracle/train_ref.py) on seeded JPEG files read by the device decoder, and rotated and
mirrored warps against cv2.warpAffine."""
import hashlib
import os
import random

import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import train_data
from centerpose_b200.coco_eval import gt_table
from centerpose_b200.config import default_cfg
from centerpose_b200.image import get_affine_transform
from oracle import train_ref
from tests.train_cases import CASES, case_cfg, dataset, seeded_case

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_batches.npz")
SPARSE = ["wh", "reg", "ind", "reg_mask", "hps", "hps_mask", "hp_offset", "hp_ind", "hp_mask"]
KEYS = ["input", "hm", "reg_mask", "ind", "wh", "hps", "hps_mask", "reg", "hm_hp", "hp_offset", "hp_ind", "hp_mask"]
DTYPES = {"input": torch.float32, "hm": torch.float32, "hm_hp": torch.float32, "wh": torch.float32,
          "reg": torch.float32, "ind": torch.int64, "reg_mask": torch.uint8, "hps": torch.float32,
          "hps_mask": torch.uint8, "hp_offset": torch.float32, "hp_ind": torch.int64, "hp_mask": torch.int64}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _batch(cfg, ds, images, np_seed, py_seed):
    tr = train_data.TrainData(cfg, ds)
    np.random.seed(np_seed)
    random.seed(py_seed)
    out = tr.batch(images, [im["id"] for im in ds["images"]])
    return {k: v.cpu().numpy() for k, v in out.items()}, out


@pytest.mark.parametrize("ci", range(len(CASES)), ids=[c[0] for c in CASES])
def test_batch_matches_golden(ci):
    from oracle.make_golden_val import image
    gold = np.load(GOLD)
    name, settings, res, np_seed, py_seed = CASES[ci]
    cfg = case_cfg(default_cfg("dla_34"), settings, res)
    ds = dataset(name)
    pix = [image(1000 * ci + im["id"], im["height"], im["width"]) for im in ds["images"]]
    assert _sha(np.concatenate([p.reshape(-1) for p in pix])) == str(gold[name + "/img_sha"])
    got, dev = _batch(cfg, ds, pix, np_seed, py_seed)
    assert list(got) == KEYS
    B, R = len(pix), res // 4
    for k in KEYS:
        assert dev[k].is_cuda and dev[k].dtype == DTYPES[k] and dev[k].shape[0] == B, k
    assert got["input"].shape == (B, 3, res, res) and got["hm"].shape == (B, 1, R, R)
    for n in range(B):
        key = "%s/%d/" % (name, n)
        for k in SPARSE:
            want = gold[key + k]
            assert got[k][n].dtype == want.dtype and np.array_equal(got[k][n].view(np.uint8), want.view(np.uint8)), \
                (key, k)
        for k in ("input", "hm", "hm_hp"):
            assert _sha(got[k][n]) == str(gold[key + k + "_sha"]), (key, k)


def test_batch_gates_keys_as_the_reference():
    ds = dataset("small_flip")
    cfg = case_cfg(default_cfg("dla_34"), {}, 128)
    cfg.LOSS.REG_OFFSET, cfg.LOSS.HM_HP, cfg.LOSS.REG_HP_OFFSET = False, False, False
    rng = np.random.default_rng(0)
    pix = [rng.integers(0, 256, (im["height"], im["width"], 3), dtype=np.uint8) for im in ds["images"]]
    got, _ = _batch(cfg, ds, pix, 0, 0)
    assert list(got) == ["input", "hm", "reg_mask", "ind", "wh", "hps", "hps_mask"]


# settings, INPUT_RES: the wider seeded matrix through the device JPEG decoder
MATRIX = [({}, 128), ({"AUG_ROT": 1., "ROTATE": 30.}, 128), ({"RANDOM_CROP": False, "AUG_ROT": 0.5, "ROTATE": 40.}, 256),
          ({"NO_COLOR_AUG": True, "FLIP": 1.}, 96), ({"RANDOM_CROP": False, "FLIP": 0.}, 160)]


@pytest.mark.parametrize("mi", range(len(MATRIX)))
def test_batch_matches_oracle_on_jpeg_files(tmp_path, mi):
    from oracle.make_golden_val import image
    settings, res = MATRIX[mi]
    cfg = case_cfg(default_cfg("dla_34"), settings, res)
    ds = seeded_case(100 + mi, 10, lo=60, hi=900)
    paths = []
    for im in ds["images"]:
        p = str(tmp_path / ("%d.jpg" % im["id"]))
        cv2.imwrite(p, image(5000 + 10 * mi + im["id"], im["height"], im["width"]), [cv2.IMWRITE_JPEG_QUALITY, 90])
        paths.append(p)
    got, _ = _batch(cfg, ds, paths, 40 + mi, 50 + mi)
    draws = train_data.TrainDraws(cfg)
    np.random.seed(40 + mi)
    random.seed(50 + mi)
    R = res // 4
    for n, (im, path) in enumerate(zip(ds["images"], paths)):
        p = draws.draw(im["height"], im["width"])
        p["trans_input"] = get_affine_transform(p["c"], p["s"], p["rot"], [res, res])
        anns = [a for a in ds["annotations"] if a["image_id"] == im["id"]]
        want = train_ref.targets(gt_table(anns), im["width"], p["flip"], p["rot"],
                                 get_affine_transform(p["c"], p["s"], 0, [R, R]),
                                 get_affine_transform(p["c"], p["s"], p["rot"], [R, R]), R)
        want["input"] = train_ref.inputs(cv2.imread(path), p, res, cfg.DATASET.MEAN, cfg.DATASET.STD)
        for k in KEYS:
            a, b = np.ascontiguousarray(got[k][n]), np.ascontiguousarray(want[k])
            assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8)), (mi, n, k)


def test_rotated_and_mirrored_warps_match_cv2():
    """NO_COLOR_AUG: the input is cv2.warpAffine of img or img[:, ::-1] with trans_input, normalised."""
    ds = seeded_case(200, 12, lo=50, hi=700, people=(0, 3))
    cfg = case_cfg(default_cfg("dla_34"), {"AUG_ROT": 1., "ROTATE": 45., "NO_COLOR_AUG": True, "RANDOM_CROP": False},
                   192)
    rng = np.random.default_rng(3)
    pix = [rng.integers(0, 256, (im["height"], im["width"], 3), dtype=np.uint8) for im in ds["images"]]
    got, _ = _batch(cfg, ds, pix, 7, 8)
    draws = train_data.TrainDraws(cfg)
    np.random.seed(7)
    random.seed(8)
    mean, std = np.float32(cfg.DATASET.MEAN), np.float32(cfg.DATASET.STD)
    n_rot = 0
    for n, im in enumerate(ds["images"]):
        p = draws.draw(im["height"], im["width"])
        n_rot += p["rot"] != 0
        src = np.ascontiguousarray(pix[n][:, ::-1] if p["flip"] else pix[n])
        warped = cv2.warpAffine(src, get_affine_transform(p["c"], p["s"], p["rot"], [192, 192]), (192, 192),
                                flags=cv2.INTER_LINEAR)
        want = ((warped.astype(np.float32) / np.float32(255.) - mean) / std).transpose(2, 0, 1)
        assert np.array_equal(got["input"][n].view(np.uint32), np.ascontiguousarray(want).view(np.uint32)), n
    assert n_rot == len(ds["images"])

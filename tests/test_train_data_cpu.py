"""CPU tests of the training batches' host side and checker: the numpy restatement (oracle/train_ref.py) and the host
draws (train_data.TrainDraws) against the reference's __getitem__ (tests/golden/train_batches.npz), the grey rule
against cv2, the pairwise mean and its device summation plan against np.mean, the lighting vector against np.dot, the
device table layout and the refused settings."""
import hashlib
import os
import random

import cv2
import numpy as np
import pytest

from centerpose_b200 import train_data
from centerpose_b200.config import default_cfg
from oracle import train_ref
from tests.train_cases import CASES, case_cfg, dataset

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_batches.npz")
SPARSE = ["wh", "reg", "ind", "reg_mask", "hps", "hps_mask", "hp_offset", "hp_ind", "hp_mask"]


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("ci", range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_matches_golden(gold, ci):
    from oracle.make_golden_train import pixels, restated
    name, settings, res, np_seed, py_seed = CASES[ci]
    cfg = case_cfg(default_cfg("dla_34"), settings, res)
    ds = dataset(name)
    pix = pixels(ci, ds)
    assert _sha(np.concatenate([pix[im["id"]].reshape(-1) for im in ds["images"]])) == str(gold[name + "/img_sha"])
    for n, (tg, p) in enumerate(restated(ds, pix, cfg, np_seed, py_seed)):
        key = "%s/%d/" % (name, n)
        for k in SPARSE:
            want = gold[key + k]
            assert tg[k].dtype == want.dtype and np.array_equal(tg[k].view(np.uint8), want.view(np.uint8)), (key, k)
        for k in ("input", "hm", "hm_hp"):
            assert _sha(tg[k]) == str(gold[key + k + "_sha"]), (key, k)


@pytest.mark.parametrize("ci", range(len(CASES)), ids=[c[0] for c in CASES])
def test_draws_match_reference(gold, ci):
    """c, s, rot, the flip, the shuffled order, the alphas and the lighting vector, image after image."""
    name, settings, res, np_seed, py_seed = CASES[ci]
    draws = train_data.TrainDraws(case_cfg(default_cfg("dla_34"), settings, res))
    np.random.seed(np_seed)
    random.seed(py_seed)
    for n, im in enumerate(dataset(name)["images"]):
        p = draws.draw(im["height"], im["width"])
        key = "%s/%d/" % (name, n)
        assert np.array_equal(p["c"].view(np.uint32), gold[key + "c"].view(np.uint32))
        assert float(p["s"]) == float(gold[key + "s"]) and float(p["rot"]) == float(gold[key + "rot"])
        assert bool(p["flip"]) == bool(gold[key + "flip"]) and p["color"] == bool(gold[key + "color"])
        if p["color"]:
            assert list(p["order"]) == gold[key + "order"].tolist()
            assert np.array_equal(np.float64(p["alpha"]), gold[key + "alpha"])
            assert np.array_equal(p["light"].view(np.uint64), gold[key + "light"].view(np.uint64))


def test_golden_covers_the_issue_cases(gold):
    names = [c[0] for c in CASES]
    rot = [bool(float(gold["%s/%d/rot" % (c, n)]) != 0) for c in names for n in range(8) if "%s/%d/rot" % (c, n) in gold]
    flip = [bool(gold["%s/%d/flip" % (c, n)]) for c in names for n in range(8) if "%s/%d/flip" % (c, n) in gold]
    assert any(rot) and not all(rot) and any(flip) and not all(flip)
    assert {c[2] for c in CASES} == {128, 512}
    assert {bool(c[1].get("RANDOM_CROP", True)) for c in CASES} == {True, False}
    assert {bool(c[1].get("NO_COLOR_AUG", False)) for c in CASES} == {True, False}


@pytest.mark.parametrize("S", range(96, 513, 32))
def test_grey_rule_and_pairwise_mean(S):
    rng = np.random.default_rng(S)
    x = rng.integers(0, 256, (S, S, 3), dtype=np.uint8).astype(np.float32) / np.float32(255.)
    g = train_ref.grey(x)
    assert np.array_equal(g.view(np.uint32), cv2.cvtColor(x, cv2.COLOR_BGR2GRAY).view(np.uint32))
    m = train_ref.mean(g)
    assert m.view(np.uint32) == g.mean().view(np.uint32)
    # the device's summation plan, evaluated as the mean kernel evaluates it
    plan = train_data.mean_plan(S * S)
    L, D = int(plan[0]), int(plan[1])
    begin, level = plan[2:3 + L], plan[3 + L:4 + L + D]
    node = plan[4 + L + D:].reshape(-1, 2)
    a = g.reshape(-1)
    slot = np.zeros(L + len(node), np.float32)
    for i in range(L):
        leaf = a[begin[i]:begin[i + 1]]
        assert len(leaf) % 8 == 0 and 64 <= len(leaf) <= 128
        slot[i] = train_ref.pairwise_sum(leaf)
    for d in range(D):
        for k in range(level[d], level[d + 1]):
            assert node[k].max() < L + k
            slot[L + k] = slot[node[k, 0]] + slot[node[k, 1]]
    assert np.float32(slot[-1] / np.float32(S * S)).view(np.uint32) == g.mean().view(np.uint32)
    assert 2 * (L + len(node)) <= 2 * (S * S // 32)       # the mean kernel's shared-memory bound


def test_fmaf_is_correctly_rounded():
    from fractions import Fraction
    rng = np.random.default_rng(5)
    a, b, c = (rng.standard_normal(4000).astype(np.float32) for _ in range(3))
    got = train_ref.fmaf(a, b, c)
    for i in range(0, 4000, 7):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(v.view(np.uint32)) & 1))
        assert got[i] == best


def test_lighting_matches_np_dot():
    rng = np.random.RandomState(9)
    for _ in range(3000):
        alpha = rng.normal(scale=0.1, size=(3,))
        want = np.dot(train_data.EIG_VEC, train_data.EIG_VAL * alpha)
        assert np.array_equal(train_data.lighting(alpha), want)


def test_table_layout():
    t = train_data.TRAIN_IMAGE
    assert t.itemsize == 240
    want = {"offset": 0, "h": 8, "w": 12, "flip": 16, "rot": 20, "color": 24, "order": 28, "gt_begin": 40,
            "gt_count": 44, "alpha": 48, "beta": 60, "light": 72, "trans_input": 96, "trans_output": 144,
            "trans_output_rot": 192}
    assert {k: t.fields[k][1] for k in want} == want
    table = np.zeros(2, t)
    row = table[1]
    row["h"] = 7
    assert table["h"].tolist() == [0, 7]


def test_get_border_halves_for_small_images():
    assert train_data.get_border(128, 640) == 128
    assert train_data.get_border(128, 255) == 64
    assert train_data.get_border(128, 120) == 32
    assert train_data.get_border(128, 64) == 16


@pytest.mark.parametrize("section,key,value", [("LOSS", "MSE_LOSS", True), ("LOSS", "DENSE_HP", True),
                                               ("LOSS", "REG_LOSS", "sl1"), ("MODEL", "NUM_STACKS", 2),
                                               ("MODEL", "OUTPUT_RES", 64), (None, "DEBUG", 1)])
def test_refused_settings(section, key, value):
    cfg = default_cfg("dla_34")
    if section is None:
        cfg[key] = value
    else:
        cfg[section][key] = value
    with pytest.raises(NotImplementedError):
        train_data.check_cfg(cfg)

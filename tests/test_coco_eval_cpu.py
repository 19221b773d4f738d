"""CPU tests of the COCO keypoint evaluation: the numpy restatement of pycocotools (oracle/cocoeval_ref.py) on
hand-computed cases, the '{:.2f}' rounding identity the kernel uses, a model of the kernel's OKS summation order
against np.sum, the host tables of centerpose_b200/coco_eval.py, and the oracle against pycocotools itself when it is
importable."""
import math
from fractions import Fraction

import numpy as np
import pytest

from centerpose_b200 import coco_eval
from centerpose_b200.coco_format import convert_eval_format
from oracle import cocoeval_ref
from tests.coco_eval_cases import check_margins, make_case

SIGMAS = coco_eval.KPT_OKS_SIGMAS


def _gt_ann(ann_id, image_id, kx, ky, v=None, area=10000.0, iscrowd=0, num_keypoints=None):
    v = np.full(17, 2) if v is None else np.asarray(v)
    return {"id": ann_id, "image_id": image_id, "category_id": 1, "iscrowd": iscrowd, "area": area,
            "num_keypoints": int((v > 0).sum()) if num_keypoints is None else num_keypoints,
            "bbox": [float(np.min(kx)), float(np.min(ky)), 100.0, 100.0],
            "keypoints": np.stack([kx, ky, v], 1).reshape(-1).tolist()}


def _dataset(anns, image_ids):
    return {"images": [{"id": i} for i in image_ids], "annotations": anns, "categories": [{"id": 1, "name": "person"}]}


def _row(kx, ky, score, box=(0.0, 0.0, 100.0, 100.0)):
    r = np.zeros(56, np.float32)
    r[0:4] = box
    r[4] = score
    r[5:39:2], r[6:39:2] = kx, ky
    return r


def _run(gt, results, img_ids=None):
    return cocoeval_ref.evaluate(gt, convert_eval_format(results), img_ids, out=None)


def _pose(rng, cx=200.0, cy=200.0):
    return np.rint(cx + rng.uniform(-40, 40, 17)), np.rint(cy + rng.uniform(-40, 40, 17))


def _offset_for_oks(target, area):
    """The x offset d applied to every joint that gives OKS = target: exp(-d^2 / vars / (area + eps) / 2) averaged."""
    from scipy.optimize import brentq
    vars_ = (SIGMAS * 2) ** 2
    f = lambda d: np.mean(np.exp(-(d * d) / vars_ / (area + np.spacing(1)) / 2)) - target
    return brentq(f, 0.0, 100.0)


# ---- the oracle on hand-computed cases ----

def test_perfect_detections_give_one_and_empty_ranges_minus_one():
    rng = np.random.default_rng(0)
    anns, res = [], {}
    for i in range(1, 4):
        kx, ky = _pose(rng)
        anns.append(_gt_ann(i, i, kx, ky, area=2000.0))          # medium only
        res[i] = {1: np.stack([_row(kx, ky, 0.9)])}
    E = _run(_dataset(anns, [1, 2, 3]), res)
    np.testing.assert_array_equal(E.stats[[0, 1, 2, 3, 5, 6, 7, 8]], 1.0)
    assert E.stats[4] == -1 and E.stats[9] == -1                  # no 'large' ground truth
    assert np.all(E.eval["precision"][:, :, 0, 2, 0] == -1)


def test_oks_near_072_gives_ap50_one_ap75_zero():
    rng = np.random.default_rng(1)
    area = 4000.0
    d = _offset_for_oks(0.72, area)
    anns, res = [], {}
    for i in range(1, 3):                                         # two ground truths
        kx, ky = _pose(rng)
        anns.append(_gt_ann(i, i, kx, ky, area=area))
        res[i] = {1: np.stack([_row(kx + d, ky, 0.5)])}
    E = _run(_dataset(anns, [1, 2]), res)
    oks = [E.ious[i, 1][0, 0] for i in (1, 2)]
    assert all(abs(o - 0.72) < 1e-3 for o in oks)
    assert E.stats[1] == 1.0 and E.stats[2] == 0.0
    assert E.stats[0] == 0.5                                      # 5 of 10 thresholds pass, each with AP 1 or 0
    # one ground truth: spacing(1) makes the first precision 1 / (1 + 2^-52), not 1
    E1 = _run(_dataset(anns[:1], [1]), {1: res[1]})
    assert E1.eval["precision"][0, 0, 0, 0, 0] == 1.0 / (1.0 + np.spacing(1))
    assert E1.eval["precision"][0, 0, 0, 0, 0] < 1.0


def test_crowd_ground_truth_is_matched_again_and_ignored():
    rng = np.random.default_rng(2)
    kx, ky = _pose(rng)
    crowd = _gt_ann(1, 1, kx, ky, iscrowd=1)
    # two detections on the crowd: both match it (a crowd can be matched again) and both are ignored
    E = _run(_dataset([crowd], [1]), {1: {1: np.stack([_row(kx, ky, 0.9), _row(kx, ky, 0.8)])}})
    ev = E.evalImgs[0]
    assert np.all(ev["dtMatches"] == 1) and np.all(ev["dtIgnore"])
    assert E.stats[0] == -1                                       # no ground truth that counts


def test_num_keypoints_zero_is_ignored_whatever_its_ignore_field():
    rng = np.random.default_rng(3)
    kx, ky = _pose(rng)
    g0 = _gt_ann(1, 1, kx, ky)
    g1 = _gt_ann(2, 1, kx + 300, ky, num_keypoints=0)
    g0["ignore"] = 1                                              # overwritten by _prepare
    E = _run(_dataset([g0, g1], [1]), {1: {1: np.stack([_row(kx, ky, 0.9)])}})
    assert list(E.evalImgs[0]["gtIgnore"]) == [0, 1]
    assert E.stats[5] == 1.0 and abs(E.stats[0] - 1.0) < 1e-12     # one ground truth: precision 1 / (1 + 2^-52)


def test_ground_truth_id_zero_counts_as_unmatched():
    rng = np.random.default_rng(4)
    kx, ky = _pose(rng)
    E = _run(_dataset([_gt_ann(0, 1, kx, ky)], [1]), {1: {1: np.stack([_row(kx, ky, 0.9)])}})
    assert np.all(E.evalImgs[0]["dtMatches"] == 0)                # matched, but to id 0
    assert E.stats[0] == 0.0 and E.stats[5] == 0.0


def test_later_ground_truth_wins_an_oks_tie_and_ignored_ones_come_last():
    rng = np.random.default_rng(5)
    kx, ky = _pose(rng)
    a, b = _gt_ann(1, 1, kx, ky), _gt_ann(2, 1, kx, ky)          # identical: equal OKS
    E = _run(_dataset([a, b], [1]), {1: {1: np.stack([_row(kx, ky, 0.9)])}})
    assert E.evalImgs[0]["dtMatches"][0, 0] == 2
    # an ignored ground truth listed first is sorted after the others: the kept one is matched first
    c = _gt_ann(3, 1, kx, ky, iscrowd=1)
    E = _run(_dataset([c, a], [1]), {1: {1: np.stack([_row(kx, ky, 0.9)])}})
    assert E.evalImgs[0]["gtIds"] == [1, 3] and E.evalImgs[0]["dtMatches"][0, 0] == 1


def test_detections_sorted_stably_nan_last_and_cut_to_20():
    rng = np.random.default_rng(6)
    kx, ky = _pose(rng)
    scores = [0.5, np.nan, -0.001, 0.0, 0.5] + [0.3] * 30
    rows = np.stack([_row(kx + k, ky, s) for k, s in enumerate(scores)])
    E = _run(_dataset([_gt_ann(1, 1, kx, ky)], [1]), {1: {1: rows}})
    ev = E.evalImgs[0]
    assert ev["dtIds"][:2] == [1, 5] and len(ev["dtIds"]) == 20   # the 0.5 tie in results order
    assert 2 not in ev["dtIds"]                                   # NaN sorts last and is cut
    sc = [convert_eval_format({1: {1: rows}})[k]["score"] for k in (2, 3)]
    assert math.copysign(1, sc[0]) == -1 and sc[0] == sc[1] == 0.0    # -0.0 ties 0.0


def test_no_visible_joint_uses_the_box_distance():
    kx, ky = np.zeros(17), np.zeros(17)
    g = _gt_ann(1, 1, kx, ky, v=np.zeros(17), num_keypoints=3)
    g["bbox"] = [100.0, 100.0, 50.0, 50.0]
    inside = np.full(17, 120.0)                                   # inside the box three times the size: OKS 1
    E = _run(_dataset([g], [1]), {1: {1: np.stack([_row(inside, inside, 0.9)])}})
    assert E.ious[1, 1][0, 0] == 1.0
    far = np.full(17, 210.0)                                      # 10 px beyond x1 = y1 = 100 + 2 * 50
    E = _run(_dataset([g], [1]), {1: {1: np.stack([_row(far, far, 0.9)])}})
    e = (10.0 ** 2 + 10.0 ** 2) / ((SIGMAS * 2) ** 2) / (g["area"] + np.spacing(1)) / 2
    assert E.ious[1, 1][0, 0] == np.sum(np.exp(-e)) / 17


def test_loadres_area_from_the_formatted_box():
    rng = np.random.default_rng(7)
    kx, ky = _pose(rng)
    dets = convert_eval_format({1: {1: np.stack([_row(kx, ky, 0.9, box=(10.004, 20.0, 60.126, 70.5))])}})
    res = cocoeval_ref.COCO(_dataset([_gt_ann(1, 1, kx, ky)], [1])).loadRes(dets)
    ann = res.anns[1]
    assert ann["area"] == float("{:.2f}".format(np.float64(np.float32(60.126)) - np.float64(np.float32(10.004)))) * 50.5
    # results without a bbox take loadRes' keypoints branch: the keypoints' extent
    nobox = [{k: v for k, v in d.items() if k != "bbox"} for d in dets]
    ann = cocoeval_ref.COCO(_dataset([], [1])).loadRes(nobox).anns[1]
    x, y = ann["keypoints"][0::3], ann["keypoints"][1::3]
    assert ann["area"] == (max(x) - min(x)) * (max(y) - min(y))


def test_loadres_refusals():
    coco = cocoeval_ref.COCO(_dataset([], [1]))
    with pytest.raises(AssertionError):
        coco.loadRes([{"image_id": 2, "category_id": 1, "score": 1.0, "bbox": [0, 0, 1, 1], "keypoints": [0] * 51}])
    with pytest.raises(IndexError):
        coco.loadRes([])


def test_summary_lines():
    gt, res = make_case(0, n_images=10, max_rows=20)
    E = _run(gt, res)
    assert E.lines[0].startswith(" Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets= 20 ] = ")
    assert E.lines[9].startswith(" Average Recall     (AR) @[ IoU=0.50:0.95 | area= large | maxDets= 20 ] = ")
    lines = []
    stats = coco_eval.summarize_arrays(E.eval["precision"], E.eval["recall"], out=lines.append)
    assert lines == E.lines and np.array_equal(stats, E.stats)


# ---- the kernel's arithmetic, modelled ----

def _round2(v):
    """The kernel's round2: v * 100 to the nearest integer, ties to even on the exact product, divided by 100."""
    p = v * 100.0
    e = float(Fraction(v) * 100 - Fraction(p))                   # the product's rounding error, exact (an FMA)
    k = float(np.rint(p))
    d = p - k
    if d == 0.5 and e > 0:
        k += 1.0
    elif d == -0.5 and e < 0:
        k -= 1.0
    return k / 100.0


def test_round2_matches_format():
    rng = np.random.default_rng(8)
    f32 = rng.uniform(-2000, 2000, 100000).astype(np.float32).astype(np.float64)
    mids = (np.floor(rng.uniform(-2000, 2000, 5000)) + rng.choice([0.125, 0.375, 0.005, 0.015, 0.995], 5000))
    mid32 = mids.astype(np.float32).astype(np.float64)
    diffs = (rng.uniform(0, 600, 20000).astype(np.float32).astype(np.float64)
             - rng.uniform(0, 600, 20000).astype(np.float32).astype(np.float64))   # the box width and height
    for v in np.concatenate([f32, mids, mid32, diffs, [0.0, -0.0, -0.001, 0.125, 2.5e-3]]):
        want = float("{:.2f}".format(v))
        got = _round2(float(v))
        assert got == want and math.copysign(1, got) == math.copysign(1, want), v
    # for a float32 x, x * 100 is exact, so rint(x * 100) / 100 is the same rounding
    np.testing.assert_array_equal(np.rint(f32 * 100) / 100, [float("{:.2f}".format(v)) for v in f32])


def _kernel_sum(a):
    n = len(a)
    if n < 8:
        s = 0.0
        for v in a:
            s += v
        return s
    r = list(a[:8])
    i = 8
    while i + 8 <= n:
        for j in range(8):
            r[j] += a[i + j]
        i += 8
    s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for v in a[i:]:
        s += v
    return s


@pytest.mark.parametrize("n", range(1, 18))
def test_kernel_summation_order_is_numpys(n):
    rng = np.random.default_rng(100 + n)
    for _ in range(500):
        a = np.exp(-rng.random(n) * rng.choice([1e-3, 1.0, 30.0]))
        assert np.sum(a) == _kernel_sum(a.tolist())


# ---- host tables ----

def test_gt_table_packing():
    kx, ky = np.arange(17.0), np.arange(17.0) + 100
    v = np.array([2, 0, 1] + [0] * 14)
    t = coco_eval.gt_table([_gt_ann(7, 1, kx, ky, v=v, area=321.5, iscrowd=1),
                            _gt_ann(0, 1, kx, ky, v=np.zeros(17), num_keypoints=0)])
    assert t.dtype.itemsize == 336
    np.testing.assert_array_equal(t[0]["x"], kx)
    np.testing.assert_array_equal(t[0]["y"], ky)
    assert t[0]["visible"] == 0b101 and t[0]["iscrowd"] == 1 and t[0]["ignore"] == 1 and t[0]["id"] == 7
    assert t[0]["area"] == 321.5 and list(t[0]["bbox"]) == [0.0, 100.0, 100.0, 100.0]
    assert t[1]["visible"] == 0 and t[1]["ignore"] == 1 and t[1]["iscrowd"] == 0 and t[1]["id"] == 0


def test_image_table_packing():
    t, n_keep, n_oks = coco_eval.image_table([5, 0, 30, 20], [(0, 2), (2, 0), (2, 3), (5, 1)])
    assert t.dtype.itemsize == 32
    assert list(t["det_begin"]) == [0, 5, 5, 35] and list(t["det_count"]) == [5, 0, 30, 20]
    assert list(t["keep_begin"]) == [0, 5, 5, 25] and n_keep == 45
    assert list(t["oks_offset"]) == [0, 10, 10, 70] and n_oks == 90
    assert list(t["gt_begin"]) == [0, 2, 2, 5] and list(t["gt_count"]) == [2, 0, 3, 1]


def test_params_are_numpys():
    p = coco_eval.params()
    assert list(p.iou_thrs) == np.linspace(.5, 0.95, 10).tolist()
    assert list(p.rec_thrs) == np.linspace(0, 1, 101).tolist()
    assert list(p.vars) == ((cocoeval_ref.Params().kpt_oks_sigmas * 2) ** 2).tolist()
    assert list(p.area_rng) == [0.0, 1e10, 1024.0, 9216.0, 9216.0, 1e10]


def test_seeded_cases_keep_their_margins():
    for seed in range(3):
        gt, res = make_case(seed)
        E = _run(gt, res)
        check_margins(E.ious)
        assert any(len(m) and np.any(np.asarray(m) == 1.0) for m in E.ious.values())


# ---- the oracle against pycocotools ----

@pytest.mark.parametrize("seed", range(4))
def test_oracle_matches_pycocotools(seed):
    pytest.importorskip("pycocotools")
    from pycocotools.coco import COCO
    from pycocotools.cocoeval import COCOeval
    import contextlib
    import copy
    import io
    gt, res = make_case(seed)
    dets = convert_eval_format(res)
    want = _run(gt, res)
    with contextlib.redirect_stdout(io.StringIO()):
        coco = COCO()
        coco.dataset = copy.deepcopy(gt)
        coco.createIndex()
        E = COCOeval(coco, coco.loadRes(copy.deepcopy(dets)), "keypoints")
        E.evaluate()
        E.accumulate()
        E.summarize()
    for k in ("precision", "recall", "scores"):
        np.testing.assert_array_equal(want.eval[k], E.eval[k])
    np.testing.assert_array_equal(want.stats, E.stats)

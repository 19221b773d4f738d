"""GPU tests of the COCO keypoint evaluation (cpb200_coco_kp_eval / cpb200_coco_kp_oks) against the numpy
restatement of pycocotools (oracle/cocoeval_ref.py) fed by coco_format.convert_eval_format: OKS within 4 ulp,
precision / recall / scores / stats and the summary lines bit for bit, and MultiPoseDetector.run_eval end to end."""
import numpy as np
import pytest
import torch

from centerpose_b200.coco_eval import KeypointEval
from centerpose_b200.coco_format import convert_eval_format
from oracle import cocoeval_ref
from tests.coco_eval_cases import check_margins, make_case

pytestmark = pytest.mark.gpu

SEEDS = range(6)


def _oracle(gt, results, img_ids=None):
    E = cocoeval_ref.evaluate(gt, convert_eval_format(results), img_ids, out=None)
    check_margins(E.ious)
    return E


def _bit_equal(got, want, what):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, what
    np.testing.assert_array_equal(got, want, err_msg=what)          # NaN equals NaN here
    assert np.array_equal(np.signbit(got), np.signbit(want)), what + " (sign of zero)"


def _check_eval(ev, E, lines=None):
    for k in ("precision", "recall", "scores"):
        _bit_equal(ev.eval[k], E.eval[k], k)
    _bit_equal(ev.stats, E.stats, "stats")
    if lines is not None:
        assert lines == E.lines


def _forms(results, form):
    """The same results as each accepted input form."""
    if form == "dict":
        return results
    if form == "flat":
        return {k: v[1] for k, v in results.items()}
    if form == "lists":
        return {k: v[1].tolist() for k, v in results.items()}
    if form == "cuda":
        return (list(results), [torch.from_numpy(v[1]).cuda() for v in results.values()])
    return (list(results), [v[1] for v in results.values()])


@pytest.mark.parametrize("seed", SEEDS)
def test_oks_within_4_ulp(seed):
    gt, res = make_case(seed)
    E = _oracle(gt, res)
    got = KeypointEval(gt).oks(res)
    n = 0
    for (image_id, _), want in E.ious.items():
        want = np.asarray(want, np.float64)
        g = got[image_id]
        if want.size == 0:
            assert g.size == 0
            continue
        assert g.shape == want.shape
        assert np.array_equal(np.isnan(g), np.isnan(want))
        f = ~np.isnan(want)
        ulp = np.maximum(np.spacing(np.abs(want[f])), np.spacing(np.abs(g[f])))
        assert np.all(np.abs(g[f] - want[f]) <= 4 * ulp), image_id
        n += want.size
    assert n > 100


@pytest.mark.parametrize("seed,form", [(s, f) for s, f in zip(SEEDS, ["dict", "flat", "pairs", "cuda", "lists", "dict"])])
def test_eval_bit_equal_to_oracle(seed, form, capsys):
    gt, res = make_case(seed)
    E = _oracle(gt, res)
    ev = KeypointEval(gt)
    stats = ev.evaluate(_forms(res, form))
    _bit_equal(stats, E.stats, "returned stats")
    capsys.readouterr()
    ev.summarize()
    _check_eval(ev, E, capsys.readouterr().out.splitlines())


def test_eval_img_ids_subset_and_reuse():
    gt, res = make_case(7)
    ev = KeypointEval(gt)
    ids = sorted(img["id"] for img in gt["images"])
    subset = ids[::3] + [ids[1], -5]                # unsorted, a duplicate, an id the ground truth lacks
    for img_ids in (subset, None, ids[1::2]):
        E = _oracle(gt, res, img_ids)
        ev.evaluate(res, img_ids=img_ids)
        _check_eval(ev, E)


def test_eval_edges_of_the_range():
    # a range with no ground truth stays -1; images with detections and no ground truth are false positives
    gt, res = make_case(3, n_images=10, max_rows=30, gts_per_image=(1, 2))
    for a in gt["annotations"]:
        a["area"] = 2000.0                          # no 'large' ground truth
    E = _oracle(gt, res)
    ev = KeypointEval(gt)
    ev.evaluate(res)
    _check_eval(ev, E)
    assert np.all(ev.eval["precision"][:, :, 0, 2, 0] == -1)


def test_eval_val2017_sized():
    gt, res = make_case(11, n_images=5000, gts_per_image=(1, 4), rows_per_image=100)
    rows = sum(len(v[1]) for v in res.values())
    assert len(gt["annotations"]) > 5000 and rows == 300000
    E = _oracle(gt, res)
    ev = KeypointEval(gt)
    ev.evaluate(res)
    _check_eval(ev, E)


def test_run_eval_end_to_end():
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle.init_recipe import conditioned_state_dict
    cfg = default_cfg("dla_34")
    det = detector_factory[cfg.TEST.TASK](cfg)
    det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
    rng = np.random.RandomState(5)
    images = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in [(256, 320), (320, 256), (256, 256)] * 2]
    ids = [11, 3, 7, 40, 2, 19]
    rows = det.run_images(images)
    # a ground truth made from perturbed rows: some matched closely, some loosely, some missed
    anns, aid = [], 1
    for image_id, r in zip(ids, rows):
        for k in range(0, 12, 2):
            kx = np.rint(r[k, 5:39:2].astype(np.float64) + rng.normal(0, 1 + k, 17))
            ky = np.rint(r[k, 6:39:2].astype(np.float64) + rng.normal(0, 1 + k, 17))
            v = np.where(rng.random_sample(17) < 0.8, 2, 0)
            w, h = float(kx.max() - kx.min() + 1), float(ky.max() - ky.min() + 1)
            anns.append({"id": aid, "image_id": image_id, "category_id": 1, "iscrowd": int(k == 10),
                         "num_keypoints": int((v > 0).sum()), "area": w * h * 0.6,
                         "bbox": [float(kx.min()), float(ky.min()), w, h],
                         "keypoints": np.stack([kx, ky, v], 1).reshape(-1).tolist()})
            aid += 1
    gt = {"images": [{"id": i} for i in ids], "annotations": anns, "categories": [{"id": 1, "name": "person"}]}
    ap = det.run_eval(images, ids, gt)
    E = cocoeval_ref.evaluate(gt, convert_eval_format({i: {1: r.tolist()} for i, r in zip(ids, rows)}), out=None)
    assert ap == E.stats[0] and ap != -1


def test_refusals():
    gt, res = make_case(2, n_images=10, max_rows=20)
    ev = KeypointEval(gt)
    image_id, r = next(iter(res.items()))
    with pytest.raises(ValueError, match="CPU tensor"):
        ev.evaluate({image_id: torch.from_numpy(r[1])})
    with pytest.raises(AssertionError, match="coco set"):
        ev.evaluate({-1: r[1]})
    with pytest.raises(IndexError):
        ev.evaluate({image_id: np.zeros((0, 56), np.float32)})
    with pytest.raises(ValueError, match="56"):
        ev.evaluate({image_id: r[1][:, :50]})
    two = dict(gt, categories=gt["categories"] + [{"id": 2, "name": "other"}])
    with pytest.raises(NotImplementedError):
        KeypointEval(two)
    dup = dict(gt, annotations=gt["annotations"] + [dict(gt["annotations"][0])])
    with pytest.raises(ValueError, match="duplicate"):
        KeypointEval(dup)

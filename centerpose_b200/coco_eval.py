"""COCO keypoint evaluation on the device: what the reference's ``dataset.run_eval`` computes
(``lib/datasets/coco_hp.py:97-107``: ``convert_eval_format``, ``COCO.loadRes``, then ``COCOeval(..., "keypoints")``'s
``evaluate`` / ``accumulate`` / ``summarize``), number for number as pycocotools 2.0.x with the default Params, without
turning the rows into Python dicts (csrc/coco_eval.cu, ``cpb200_coco_kp_eval``).

    ev = KeypointEval("person_keypoints_val2017.json")      # parsed and uploaded once
    ev.evaluate((image_ids, detector.run_images(paths)))    # -> the 10 stats; fills ev.eval and ev.stats
    ev.summarize()                                          # prints COCOeval.summarize()'s lines

The result rows are read as float32 (what ``run()`` and ``run_images`` return); the score and the 17 keypoints are
rounded as ``'{:.2f}'`` formats them, the detection's area is ``loadRes``' w * h of the formatted box (results that
carry a bbox take that branch of ``loadRes``).  ``eval['precision']`` / ``['recall']`` / ``['scores']`` come back in
one copy; ``stats`` and the summary lines are computed from them with ``COCOeval.summarize``'s numpy expressions.
"""
from __future__ import annotations

import ctypes
import json
from collections import Counter

import numpy as np
import torch

MAX_DETS = 20
JOINTS = 17
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
AREA_RNG = [[0 ** 2, 1e5 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "medium", "large"]
KPT_OKS_SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0
VARS = (KPT_OKS_SIGMAS * 2) ** 2

GT = np.dtype([("x", "<f8", JOINTS), ("y", "<f8", JOINTS), ("area", "<f8"), ("bbox", "<f8", 4), ("id", "<i8"),
               ("iscrowd", "<i4"), ("ignore", "<i4"), ("visible", "<i4"), ("pad", "<i4")])
IMAGE = np.dtype([("det_begin", "<i8"), ("det_count", "<i4"), ("keep_begin", "<i4"), ("gt_begin", "<i4"),
                  ("gt_count", "<i4"), ("oks_offset", "<i8")])
assert GT.itemsize == 336 and IMAGE.itemsize == 32

T, R, A = len(IOU_THRS), len(REC_THRS), len(AREA_RNG)


class Params(ctypes.Structure):
    """``cpb200_coco_kp_params``: the numpy-computed constants, so the device compares with the same doubles."""
    _fields_ = [("iou_thrs", ctypes.c_double * T), ("rec_thrs", ctypes.c_double * R),
                ("vars", ctypes.c_double * JOINTS), ("area_rng", ctypes.c_double * (2 * A))]


def params() -> Params:
    p = Params()
    p.iou_thrs[:] = IOU_THRS.tolist()
    p.rec_thrs[:] = REC_THRS.tolist()
    p.vars[:] = VARS.tolist()
    p.area_rng[:] = [float(v) for r in AREA_RNG for v in r]
    return p


def _dataset(gt):
    if isinstance(gt, str):
        with open(gt) as f:
            return json.load(f)
    if isinstance(gt, dict):
        return gt
    if isinstance(getattr(gt, "dataset", None), dict):
        return gt.dataset
    raise TypeError("KeypointEval: gt must be a path, a COCO-format dict or an object with a .dataset dict, got %s"
                    % type(gt).__name__)


def gt_table(anns):
    """The ``cpb200_coco_kp_gt`` rows of ``anns`` (COCO annotation dicts) in order; ``ignore`` as ``_prepare`` sets
    it (``iscrowd or num_keypoints == 0``, any ``ignore`` field of the annotation overwritten)."""
    t = np.zeros(len(anns), GT)
    for n, a in enumerate(anns):
        kp = np.asarray(a["keypoints"], np.float64).reshape(JOINTS, 3)
        crowd = a.get("iscrowd", 0)
        t[n]["x"], t[n]["y"] = kp[:, 0], kp[:, 1]
        t[n]["area"] = a["area"]
        t[n]["bbox"] = a["bbox"]
        t[n]["id"] = a["id"]
        t[n]["iscrowd"] = int(crowd)
        t[n]["ignore"] = bool(crowd) or a["num_keypoints"] == 0
        t[n]["visible"] = int(np.dot(kp[:, 2] > 0, 1 << np.arange(JOINTS)))
    return t


def image_table(det_counts, gt_ranges):
    """The ``cpb200_coco_kp_image`` rows for images with ``det_counts[i]`` consecutive rows each (packed from row 0)
    and ground truths ``gt_ranges[i] = (begin, count)``.  Returns ``(table, n_keep, n_oks)``."""
    n = len(det_counts)
    t = np.zeros(n, IMAGE)
    dc = np.asarray(det_counts, np.int64)
    keep = np.minimum(dc, MAX_DETS)
    gr = np.asarray(gt_ranges, np.int64).reshape(n, 2)
    t["det_begin"] = np.cumsum(dc) - dc
    t["det_count"] = dc
    t["keep_begin"] = np.cumsum(keep) - keep
    t["gt_begin"], t["gt_count"] = gr[:, 0], gr[:, 1]
    oks = keep * gr[:, 1]
    t["oks_offset"] = np.cumsum(oks) - oks
    return t, int(keep.sum()), int(oks.sum())


def summarize_arrays(precision, recall, out=print):
    """``COCOeval.summarize`` for keypoints (``_summarizeKps``) on ``eval['precision']`` / ``['recall']``: the ten
    stats, each line passed to ``out`` (None: not printed)."""
    def _summarize(ap=1, iouThr=None, areaRng="all", maxDets=100):
        iStr = " {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}"
        titleStr = "Average Precision" if ap == 1 else "Average Recall"
        typeStr = "(AP)" if ap == 1 else "(AR)"
        iouStr = "{:0.2f}:{:0.2f}".format(IOU_THRS[0], IOU_THRS[-1]) if iouThr is None else "{:0.2f}".format(iouThr)
        aind = [i for i, aRng in enumerate(AREA_LBL) if aRng == areaRng]
        mind = [i for i, mDet in enumerate([MAX_DETS]) if mDet == maxDets]
        s = precision if ap == 1 else recall
        if iouThr is not None:
            s = s[np.where(iouThr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        if out is not None:
            out(iStr.format(titleStr, typeStr, iouStr, areaRng, maxDets, mean_s))
        return mean_s

    stats = np.zeros((10,))
    stats[0] = _summarize(1, maxDets=20)
    stats[1] = _summarize(1, maxDets=20, iouThr=.5)
    stats[2] = _summarize(1, maxDets=20, iouThr=.75)
    stats[3] = _summarize(1, maxDets=20, areaRng="medium")
    stats[4] = _summarize(1, maxDets=20, areaRng="large")
    stats[5] = _summarize(0, maxDets=20)
    stats[6] = _summarize(0, maxDets=20, iouThr=.5)
    stats[7] = _summarize(0, maxDets=20, iouThr=.75)
    stats[8] = _summarize(0, maxDets=20, areaRng="medium")
    stats[9] = _summarize(0, maxDets=20, areaRng="large")
    return stats


def _entries(results):
    """``(image_id, rows)`` pairs in results order from ``{image_id: {1: rows}}``, ``{image_id: rows}`` or
    ``(image_ids, list_of_rows)``."""
    if isinstance(results, dict):
        return [(k, v[1] if isinstance(v, dict) else v) for k, v in results.items()]
    if isinstance(results, (tuple, list)) and len(results) == 2:
        ids, rows = results
        if len(ids) != len(rows):
            raise ValueError("KeypointEval: %d image ids for %d row sets" % (len(ids), len(rows)))
        return list(zip(ids, rows))
    raise TypeError("KeypointEval: results must be {image_id: {1: rows}}, {image_id: rows} or (image_ids, rows)")


def _rows(image_id, rows, dev):
    """Image ``image_id``'s rows as a (N, 56) float32 block: a CUDA tensor on ``dev`` or a host array."""
    if isinstance(rows, torch.Tensor):
        if not rows.is_cuda:
            raise ValueError("KeypointEval: the rows of image %r are a CPU tensor; pass a numpy array or a CUDA tensor"
                             % (image_id,))
        if rows.device != dev:
            raise ValueError("KeypointEval: the rows of image %r are on %s, the ground truth on %s"
                             % (image_id, rows.device, dev))
        t = rows.reshape(-1, 56) if rows.numel() == 0 else rows
        if t.dim() != 2 or t.shape[1] != 56:
            raise ValueError("KeypointEval: the rows of image %r have shape %s, expected (N, 56)"
                             % (image_id, tuple(rows.shape)))
        return t.float().contiguous()
    a = np.asarray(rows, np.float32)
    a = a.reshape(-1, 56) if a.size == 0 else a
    if a.ndim != 2 or a.shape[1] != 56:
        raise ValueError("KeypointEval: the rows of image %r have shape %s, expected (N, 56)" % (image_id, a.shape))
    return a


class KeypointEval:
    """``COCOeval(gt, gt.loadRes(convert_eval_format(results)), "keypoints")`` on the device.  ``gt`` is a path to a
    ``person_keypoints_*.json``, its loaded dict, or an object with a ``.dataset`` dict (pycocotools' ``COCO``).  It is
    parsed and uploaded once, to ``device`` (the current CUDA device by default); every ``evaluate`` reuses it."""

    def __init__(self, gt, device=None):
        ds = _dataset(gt)
        cats = ds.get("categories", [])
        if len(cats) != 1:
            raise NotImplementedError("KeypointEval: the ground truth has %d categories; only single-category "
                                      "(person) keypoint sets are supported" % len(cats))
        self.cat_id = cats[0]["id"]
        anns = ds.get("annotations", [])
        dup = sorted(i for i, c in Counter(a["id"] for a in anns).items() if c > 1)
        if dup:
            raise ValueError("KeypointEval: duplicate annotation ids %s (COCO.loadAnns would collapse them)" % dup[:10])
        self.img_ids = sorted({img["id"] for img in ds.get("images", [])})
        per_image = {i: [] for i in self.img_ids}
        for a in anns:
            if a["category_id"] == self.cat_id and a["image_id"] in per_image:
                per_image[a["image_id"]].append(a)
        ordered, self.gt_range = [], {}
        for i in self.img_ids:
            self.gt_range[i] = (len(ordered), len(per_image[i]))
            ordered += per_image[i]
        # coco.getImgIds(imgIds, catIds): the images with an annotation of the category (crowds count), what the
        # reference's COCOHP dataset iterates
        self.cat_img_ids = [i for i in self.img_ids if per_image[i]]
        self.device = torch.device("cuda") if device is None else torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        table = gt_table(ordered)
        self.n_gts = len(table)
        self.gts = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).to(self.device) if len(table) else \
            torch.zeros(GT.itemsize, dtype=torch.uint8, device=self.device)
        self.params = params()
        self.eval = {}
        self.stats = []

    def _pack(self, results, img_ids):
        """The evaluated images (sorted), their launch table and their rows in one device buffer."""
        entries = _entries(results)
        known = set(self.gt_range)
        for image_id, _ in entries:
            if image_id not in known:
                raise AssertionError("Results do not correspond to current coco set (image id %r)" % (image_id,))
        blocks = {}
        for image_id, rows in entries:
            blocks.setdefault(image_id, []).append(_rows(image_id, rows, self.device))
        if sum(len(b) for bs in blocks.values() for b in bs) == 0:
            raise IndexError("KeypointEval: no detections (COCO.loadRes needs at least one result)")
        evaluated = [i for i in (self.img_ids if img_ids is None else np.unique(list(img_ids)).tolist()) if i in known]
        # convert_eval_format writes category 1; another ground-truth category matches none of the detections
        take = [blocks.get(i, []) if self.cat_id == 1 else [] for i in evaluated]
        table, n_keep, n_oks = image_table([sum(len(b) for b in bs) for bs in take],
                                           [self.gt_range[i] for i in evaluated])
        flat = [b for bs in take for b in bs if len(b)]
        if any(isinstance(b, torch.Tensor) for b in flat):
            rows = torch.cat([b if isinstance(b, torch.Tensor) else torch.from_numpy(b).to(self.device) for b in flat])
        elif flat:
            host = torch.from_numpy(np.concatenate(flat)).pin_memory()
            rows = host.to(self.device, non_blocking=True)
        else:
            rows = torch.zeros((1, 56), dtype=torch.float32, device=self.device)
        n_rows = int(table["det_count"].sum()) if len(table) else 0
        up = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).pin_memory().to(self.device, non_blocking=True)
        return evaluated, table, up, rows, n_rows, n_keep, n_oks

    def _workspace(self, n_images, n_rows, n_keep, n_oks):
        from . import _lib
        nb = _lib.lib().cpb200_coco_kp_eval_workspace_bytes(n_images, n_rows, self.n_gts, n_keep, n_oks)
        return torch.empty(nb, dtype=torch.uint8, device=self.device)

    def oks(self, results, img_ids=None):
        """``COCOeval.computeOks`` alone: ``{image_id: (D, G) float64 array}`` for every evaluated image, D its first
        min(N, 20) detections by score, G its ground truths in file order (``cpb200_coco_kp_oks``)."""
        from . import _lib
        evaluated, table, up, rows, n_rows, n_keep, n_oks = self._pack(results, img_ids)
        if not evaluated:
            return {}
        out = torch.empty(max(n_oks, 1), dtype=torch.float64, device=self.device)
        ws = self._workspace(len(evaluated), n_rows, n_keep, n_oks)
        with torch.cuda.device(self.device):
            st = _lib.lib().cpb200_coco_kp_oks(up.data_ptr(), len(evaluated), rows.data_ptr(), n_rows,
                                               self.gts.data_ptr(), self.n_gts, n_keep, n_oks, ctypes.byref(self.params),
                                               out.data_ptr(), ws.data_ptr(),
                                               torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(st, "coco_kp_oks")
        host = out.cpu().numpy()
        res = {}
        for i, e in zip(evaluated, table):
            d, g = min(int(e["det_count"]), MAX_DETS), int(e["gt_count"])
            res[i] = host[e["oks_offset"]:e["oks_offset"] + d * g].reshape(d, g) if d and g else np.zeros((0, 0))
        return res

    def evaluate(self, results, img_ids=None):
        """``evaluate()`` and ``accumulate()`` on ``results`` (``{image_id: {1: rows}}``, ``{image_id: rows}`` or
        ``(image_ids, list_of_rows)``; rows (N, 56) float32 arrays, lists of floats or CUDA tensors) over ``img_ids``
        (``params.imgIds``; every ground-truth image by default).  Raises as ``loadRes`` does for an image id not in
        the ground truth and for no detections at all.  Fills ``.eval`` and ``.stats``; returns ``stats``."""
        from . import _lib
        evaluated, table, up, rows, n_rows, n_keep, n_oks = self._pack(results, img_ids)
        precision = -np.ones((T, R, 1, A, 1))
        recall = -np.ones((T, 1, A, 1))
        scores = -np.ones((T, R, 1, A, 1))
        if evaluated:
            out = torch.empty(2 * T * R * A + T * A, dtype=torch.float64, device=self.device)
            ws = self._workspace(len(evaluated), n_rows, n_keep, n_oks)
            p = out.data_ptr()
            with torch.cuda.device(self.device):
                st = _lib.lib().cpb200_coco_kp_eval(up.data_ptr(), len(evaluated), rows.data_ptr(), n_rows,
                                                    self.gts.data_ptr(), self.n_gts, n_keep, n_oks,
                                                    ctypes.byref(self.params), p, p + 8 * 2 * T * R * A,
                                                    p + 8 * T * R * A, ws.data_ptr(),
                                                    torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(st, "coco_kp_eval")
            host = out.cpu().numpy()
            precision = host[:T * R * A].reshape(T, R, 1, A, 1).copy()
            scores = host[T * R * A:2 * T * R * A].reshape(T, R, 1, A, 1).copy()
            recall = host[2 * T * R * A:].reshape(T, 1, A, 1).copy()
        self.img_ids_evaluated = evaluated
        self.eval = {"counts": [T, R, 1, A, 1], "precision": precision, "recall": recall, "scores": scores}
        self.stats = summarize_arrays(precision, recall, out=None)
        return self.stats

    def summarize(self):
        """Prints ``COCOeval.summarize()``'s ten lines and returns ``stats``."""
        if not self.eval:
            raise Exception("Please run accumulate() first")
        self.stats = summarize_arrays(self.eval["precision"], self.eval["recall"])
        return self.stats
